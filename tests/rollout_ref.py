"""CPU restatement of the reference's policy roll-out (test infrastructure only): what MRT_BASE::rolloutPolicy computes, function by function, in
plain numpy around any flow map -- for the whole-body OCP the oracle's own dynamics (oracle/rbd.hpp through oracle_lib.WbOracle.flow_map), not
the kernels' phase functions.

    RungeKuttaDormandPrince5 (ODE45_OCS2)      ocs2_core/src/integration/RungeKuttaDormandPrince5.cpp:40-64 (lessWithSign), 84-227 (Stepper),
                                               263-289 (runIntegrateAdaptive), RungeKuttaDormandPrince5.h:93 (maxNumStepsRetries_ = 100)
    IntegratorBase::systemFunction             ocs2_core/src/integration/IntegratorBase.cpp:47-58 (function-call budget; a status here, not a throw)
    RolloutBase::findActiveModesTimeInterval   ocs2_oc/src/rollout/RolloutBase.cpp:44-68
    TimeTriggeredRollout::run                  ocs2_oc/src/rollout/TimeTriggeredRollout.cpp:46-116 (identity jump map, reconstructInputTrajectory)
    LinearInterpolation::timeSegment           ocs2_core/include/ocs2_core/misc/implementation/LinearInterpolation.h:69-105 (lookup::findIntervalInTimeArray)
    LinearController / FeedforwardController::computeInput   ocs2_core/src/control/LinearController.cpp:79-87, FeedforwardController.cpp:89-91
    ModeSchedule::modeAtTime                   ocs2_core/src/reference/ModeSchedule.cpp:50-53 (lookup::findIndexInTimeArray = lower_bound)
    MRT_BASE::rolloutPolicy                    ocs2_mpc/src/MRT_BASE.cpp:124-151

The controller is built from a primal solution as the shim does (include/ocs2_sqp/B200SqpSolver.h, toPrimalSolution): node k carries the input
and gain of stage src = k (the terminal node and PreEvent nodes repeat the stage before them) and bias_k = u_k - K_k x_k.  The vector arithmetic
keeps the reference's expression order (Eigen evaluates its expressions coefficient-wise, left to right)."""
from __future__ import annotations

import bisect

import numpy as np

EPS = float(np.finfo(float).eps)
WEAK_EPS = 1e-9   # numeric_traits::weakEpsilon
MAX_RETRIES = 100
OK, RETRIES, BUDGET, NONFINITE = 0, 1, 2, 3


class _Abort(Exception):
    def __init__(self, status):
        self.status = status


def less_with_sign(t1, t2, dt):
    return (t2 - t1 > EPS) if dt > 0 else (t1 - t2 > EPS)


class DormandPrince5:
    """The stepper and runIntegrateAdaptive; system(x, t) -> dxdt.  Counts accepted / rejected steps and function calls across calls of
    integrate_adaptive (one TimeTriggeredRollout::run resets them once)."""

    A = (1.0 / 5, 3.0 / 10, 4.0 / 5, 8.0 / 9)
    C1, C3, C4, C5, C6 = 35.0 / 384, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84

    def __init__(self, system, max_calls=None):
        self.system = system
        self.max_calls = max_calls
        self.accepted = self.rejected = self.calls = 0

    def f(self, x, t):
        dxdt = self.system(x, t)
        self.calls += 1
        if self.max_calls is not None and self.calls > self.max_calls:
            raise _Abort(BUDGET)
        return dxdt

    def do_step(self, x0, dxdt, t, dt):
        a2, a3, a4, a5 = self.A
        k1 = dxdt
        k2 = self.f(x0 + (dt * (1.0 / 5)) * k1, t + dt * a2)
        k3 = self.f((x0 + (dt * (3.0 / 40)) * k1) + (dt * (9.0 / 40)) * k2, t + dt * a3)
        k4 = self.f(x0 + dt * (((44.0 / 45) * k1 + (-56.0 / 15) * k2) + (32.0 / 9) * k3), t + dt * a4)
        k5 = self.f(x0 + dt * ((((19372.0 / 6561) * k1 + (-25360.0 / 2187) * k2) + (64448.0 / 6561) * k3) + (-212.0 / 729) * k4), t + dt * a5)
        k6 = self.f(x0 + dt * (((((9017.0 / 3168) * k1 + (-355.0 / 33) * k2) + (46732.0 / 5247) * k3) + (49.0 / 176) * k4) + (-5103.0 / 18656) * k5),
                    t + dt)
        x_out = x0 + dt * ((((self.C1 * k1 + self.C3 * k3) + self.C4 * k4) + self.C5 * k5) + self.C6 * k6)
        dxdt_out = self.f(x_out, t + dt)
        return x_out, dxdt_out, (k1, k3, k4, k5, k6)

    @staticmethod
    def max_error(x_old, dxdt_old, x_err, dt, abs_tol, rel_tol):
        err = np.abs(x_err / (abs_tol + rel_tol * (np.abs(x_old) + abs(dt) * np.abs(dxdt_old))))
        return float(np.max(err))   # NaN propagates

    @staticmethod
    def decrease_step(dt, error):
        return dt * max(0.9 * error ** (-1.0 / 3), 0.2)

    @staticmethod
    def increase_step(dt, error):
        if error < 0.5:
            error = max(5.0 ** -5, error)
            dt *= 0.9 * error ** (-1.0 / 5)
        return dt

    def try_step(self, x, dxdt, t, dt, abs_tol, rel_tol):
        c1, c3, c4, c5, c6 = self.C1, self.C3, self.C4, self.C5, self.C6
        dc1, dc3, dc4 = c1 - 5179.0 / 57600, c3 - 7571.0 / 16695, c4 - 393.0 / 640
        dc5, dc6, dc7 = c5 - -92097.0 / 339200, c6 - 187.0 / 2100, -1.0 / 40
        x_out, dxdt_out, (k1, k3, k4, k5, k6) = self.do_step(x, dxdt, t, dt)
        x_err = dt * (((((dc1 * k1 + dc3 * k3) + dc4 * k4) + dc5 * k5) + dc6 * k6) + dc7 * dxdt_out)
        error = self.max_error(x, dxdt, x_err, dt, abs_tol, rel_tol)
        if error > 1.0:
            self.rejected += 1
            return False, x, dxdt, t, self.decrease_step(dt, error)
        self.accepted += 1
        return True, x_out, dxdt_out, t + dt, self.increase_step(dt, error)

    def integrate_adaptive(self, x0, t0, tf, dt0, abs_tol, rel_tol, observer):
        t, dt, x = t0, dt0, np.array(x0, dtype=float)
        dxdt = self.f(x, t)
        while less_with_sign(t, tf, dt):
            observer(x, t)
            if less_with_sign(tf, t + dt, dt):
                dt = tf - t
            tries = 0
            while True:
                ok, x, dxdt, t, dt = self.try_step(x, dxdt, t, dt, abs_tol, rel_tol)
                if ok:
                    break
                tries += 1
                if tries > MAX_RETRIES:
                    raise _Abort(RETRIES)
        observer(x, t)


def integrate_adaptive(system, x0, t0, tf, dt0=0.01, abs_tol=1e-6, rel_tol=1e-3):
    """IntegratorBase::integrateAdaptive with the ODE45_OCS2 integrator -> (times, states, stepper)"""
    ts, xs = [], []
    dp = DormandPrince5(system)
    dp.integrate_adaptive(x0, t0, tf, dt0, abs_tol, rel_tol, lambda x, t: (xs.append(np.array(x)), ts.append(t)))
    return np.array(ts), np.array(xs), dp


def find_active_modes_time_interval(t0, tf, event_times):
    """events in (t0, tf]; every interval starts weakEpsilon after its switching time (a degenerate interval has first == second)"""
    ev = list(event_times)
    sw = [t0] + ev[bisect.bisect_right(ev, t0):bisect.bisect_right(ev, tf)] + [tf]
    return [(min(sw[i] + WEAK_EPS, sw[i + 1]), sw[i + 1]) for i in range(len(sw) - 1)]


def time_segment(t, times):
    """LinearInterpolation::timeSegment -> (index, alpha)"""
    n = len(times)
    if n <= 1:
        return 0, 1.0
    index = bisect.bisect_left(times, t) - 1
    last = n - 1
    if index < 0:
        return 0, 1.0
    if index < last:
        length, till = times[index + 1] - times[index], times[index + 1] - t
        if length > 2.0 * WEAK_EPS:
            return index, till / length
        return index, (0.0 if till < 0.5 * length else 1.0)
    return max(last - 1, 0), 0.0


class PlanController:
    """LinearController (K given) or FeedforwardController of one primal solution: t [n], event [n], x [n, nx], u [n-1, nu], K [n-1, nu, nx]"""

    def __init__(self, t, event, x, u, K=None):
        n = len(t)
        self.t = [float(v) for v in t]
        self.src = [min(k, n - 2) if not (event[k] == 1 and k > 0) else k - 1 for k in range(n)]
        self.u = [np.array(u[s], dtype=float) for s in self.src]
        self.K = None
        if K is not None:
            self.K = [np.array(K[s], dtype=float) for s in self.src]
            self.bias = []
            for k in range(n):   # uff = u - K x, s = u_r; s -= K_rc x_c in increasing c
                s = self.u[k].copy()
                for c in range(x.shape[1]):
                    s -= self.K[k][:, c] * x[k][c]
                self.bias.append(s)

    def compute_input(self, t, x):
        i, a = time_segment(t, self.t)
        if self.K is None:
            return a * self.u[i] + (1.0 - a) * self.u[i + 1]
        u = a * self.bias[i] + (1.0 - a) * self.bias[i + 1]
        k = a * self.K[i] + (1.0 - a) * self.K[i + 1]
        for c in range(len(x)):
            u = u + k[:, c] * x[c]
        return u


def mode_at_time(t, event_times, modes):
    return modes[bisect.bisect_left(list(event_times), t)]


def time_triggered_rollout(flow_map, controller, t0, x0, tf, event_times, abs_tol=1e-5, rel_tol=1e-3, time_step=0.015, max_steps_per_second=10000):
    """TimeTriggeredRollout::run -> dict(t, x, u, post_event_indices, accepted, rejected, calls, status)"""
    if t0 > tf:
        raise ValueError("the initial time should be less-equal to the final time")
    intervals = find_active_modes_time_interval(t0, tf, event_times)
    max_calls = int(max_steps_per_second * max(1.0, tf - t0))
    dp = DormandPrince5(lambda x, t: flow_map(x, controller.compute_input(t, x)), max_calls)
    ts, xs, post = [], [], []
    begin = np.array(x0, dtype=float)
    status = OK
    try:
        for i, (a, b) in enumerate(intervals):
            if a < b:
                dp.integrate_adaptive(begin, a, b, time_step, abs_tol, rel_tol, lambda x, t: (xs.append(np.array(x)), ts.append(t)))
            else:
                ts.append(b)
                xs.append(begin.copy())
            if i < len(intervals) - 1:
                post.append(len(xs))
                begin = xs[-1].copy()   # identity jump map
    except _Abort as e:
        status = e.status
    us = [controller.compute_input(t, x) for t, x in zip(ts, xs)] if status == OK else []
    if status == OK and not (np.all(np.isfinite(xs[-1])) and np.all(np.isfinite(us[-1]))):
        status = NONFINITE
    return dict(t=np.array(ts), x=np.array(xs), u=np.array(us), post_event_indices=post, accepted=dp.accepted, rejected=dp.rejected, calls=dp.calls,
                status=status)


def plan_event_times_and_modes(t, event, contact):
    """the plan's PreEvent node times and the mode (0 FLY, 1 RF, 2 LF, 3 STANCE) of every segment, read from the contact flags of its first node"""
    ev = [float(t[k]) for k in range(len(t)) if event[k] == 1]
    starts = [0] + [k + 1 for k in range(len(t)) if event[k] == 1]
    modes = [2 * int(contact[k][0]) + int(contact[k][1]) for k in starts]
    return ev, modes


def rollout_policy(flow_map, plan, t, duration, x, K=None, **settings):
    """MRT_BASE::rolloutPolicy on one instance.  plan: dict(t_nodes, node_event, contact_flags, x [n, nx], u [n-1, nu]); K [n-1, nu, nx] or None.
    -> dict(x, u, mode, accepted, rejected, calls, status, t_end)"""
    ev, modes = plan_event_times_and_modes(plan["t_nodes"], plan["node_event"], plan["contact_flags"])
    ctrl = PlanController(plan["t_nodes"], plan["node_event"], plan["x"], plan["u"], K)
    tf = t + duration
    r = time_triggered_rollout(flow_map, ctrl, t, x, tf, ev, **settings)
    out = dict(accepted=r["accepted"], rejected=r["rejected"], calls=r["calls"], status=r["status"], mode=mode_at_time(tf, ev, modes))
    if r["status"] == OK or r["status"] == NONFINITE:
        out.update(x=r["x"][-1], u=r["u"][-1], t_end=r["t"][-1])
    return out
