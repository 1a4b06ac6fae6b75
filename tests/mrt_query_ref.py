"""numpy restatement of the MRT-side queries: MPC_MRT_Interface::getValueFunction (SqpSolver::getValueFunction, SqpSolver.cpp:172-191) and
getLinearFeedbackGain at one time t, over one instance's plan.  LinearInterpolation::timeSegment over the node times, entry-wise interpolation
alpha a + (1 - alpha) b, the re-centring dfdx += dfdxx x one column at a time in increasing order, and the node -> stage map of
toPrimalSolution for the gains.  Every numpy operation here is one rounded IEEE operation per entry, in the order of the C++ host layer."""
from __future__ import annotations

import numpy as np

WEAK_EPS = 1e-9   # numeric_traits::weakEpsilon


def time_segment(T, t):
    """LinearInterpolation::timeSegment -> (index, alpha)"""
    n = len(T)
    if n <= 1:
        return 0, 1.0
    index = int(np.searchsorted(np.asarray(T), t, side="left")) - 1   # std::lower_bound
    last = n - 1
    if index < 0:
        return 0, 1.0
    if index < last:
        length, till = float(T[index + 1]) - float(T[index]), float(T[index + 1]) - t
        return index, (till / length if length > 2.0 * WEAK_EPS else (0.0 if till < 0.5 * length else 1.0))
    return max(last - 1, 0), 0.0


def source(event, n, k):
    """the stage whose input and gain node k carries (toPrimalSolution)"""
    src = k if k + 1 < n else n - 2
    if event[k] == 1 and k > 0:
        src = k - 1
    return src


def query(t, t_nodes, node_event, P=None, p=None, K=None, x=None):
    """P [n, nx, nx], p [n, nx], K [n-1, nu, nx] (natural orientation), x [nx] -> {dfdxx [nx, nx], dfdx [nx], K [nu, nx]} for what was given
    (dfdx needs P, p and x)"""
    idx, a = time_segment(t_nodes, t)
    b = 1.0 - a
    out = {}
    if P is not None:
        dfdxx = a * np.asarray(P[idx]) + b * np.asarray(P[idx + 1])
        out["dfdxx"] = dfdxx
        if p is not None and x is not None:
            v = a * np.asarray(p[idx]) + b * np.asarray(p[idx + 1])
            for c in range(len(x)):
                v = v + dfdxx[:, c] * x[c]
            out["dfdx"] = v
    if K is not None:
        n = len(t_nodes)
        out["K"] = a * np.asarray(K[source(node_event, n, idx)]) + b * np.asarray(K[source(node_event, n, idx + 1)])
    return out
