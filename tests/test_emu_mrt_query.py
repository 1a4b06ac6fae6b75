"""The MRT queries' arithmetic (wb_query.cuh: mrtQuery, run on the CPU harness with 24 thread slices visited in reverse) against the numpy
restatement of getValueFunction / getLinearFeedbackGain (mrt_query_ref.py), on whole-body (58-wide) and centroidal (35 of 58) device
layouts whose padding is NaN: t before the first node, on every node, inside segments and past the last node; PreEvent / PostEvent pairs
of zero length and segments shorter than 2 weakEpsilon; two-node plans; PreEvent nodes and the terminal node taking the gain of the stage
before them.  Agreement to 1e-15 relative.  And the new C entry points are exported and never compute without a device."""
import ctypes as C

import numpy as np
import pytest

import mrt_query_ref as ref
from emu_build import build
from wb_humanoid_mpc_b200 import lib as _l

NX, NU = 58, 35
FAMS = {"wb": 58, "cen": 35}
NEW_SYMBOLS = ["b200sqp_mrt_query", "b200sqp_fleet_mrt_query", "b200sqp_mrt_query_dev", "b200sqp_fleet_mrt_query_dev",
               "b200sqp_fleet_download_value_function"]
_LIB = []


def emu():
    if not _LIB:
        _LIB.append(C.CDLL(str(build("mrt_query_emu.cu", "libmrtqueryemu.so"))))
    return _LIB[0]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def plan(n_base=12, seed=0):
    """node times on a 0.02 grid from 0.3 with a zero-length PreEvent / PostEvent pair, a pair 1.5e-9 apart (shorter than 2 weakEpsilon) and a
    PreEvent right before the terminal node; event codes 1 PreEvent, 2 PostEvent"""
    t, ev = [], []
    for k in range(n_base):
        tk = 0.3 + 0.02 * k
        if k == 4:
            t += [tk, tk]
            ev += [1, 2]
        elif k == 8:
            t += [tk, tk + 1.5e-9]
            ev += [1, 2]
        else:
            t.append(tk)
            ev.append(0)
    t.append(t[-1] + 0.013)   # a PreEvent node second to last
    ev[-1] = 1
    ev.append(0)
    return np.array(t), np.array(ev, dtype=np.uint8)


def device_blocks(n, sx, rng, fill=np.nan):
    """P [n][NX*NX], p [n][NX], K [n-1][NU*NX] in the device layout (column-major, the padding of a 35-wide state set to fill)"""
    P = np.full((n, NX, NX), fill)
    Pn = rng.normal(size=(n, sx, sx))
    P[:, :sx, :sx] = Pn + np.swapaxes(Pn, 1, 2)
    p = np.full((n, NX), fill)
    p[:, :sx] = rng.normal(size=(n, sx)) * 10.0
    K = np.full((n - 1, NU, NX), fill)
    K[:, :, :sx] = rng.normal(size=(n - 1, NU, sx))
    dev = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(a.shape[0], -1)   # natural -> column-major rows
    return dev(P), np.ascontiguousarray(p), dev(K), P[:, :sx, :sx].copy(), p[:, :sx].copy(), K[:, :, :sx].copy()


def run(t_nodes, event, Pd, pd, Kd, sx, tq, x, want=("dfdxx", "dfdx", "K")):
    n = len(t_nodes)
    o = {k: np.full(s, -7.0) for k, s in (("dfdxx", sx * sx), ("dfdx", sx), ("K", NU * sx)) if k in want}
    idx = emu().emu_mrt_query(C.c_int(n), _p(np.ascontiguousarray(t_nodes)), event.ctypes.data_as(C.POINTER(C.c_uint8)), _p(Kd), _p(Pd), _p(pd),
                              C.c_int(sx), C.c_double(tq), _p(None if x is None else np.ascontiguousarray(x)), _p(o.get("dfdxx")), _p(o.get("dfdx")),
                              _p(o.get("K")))
    if "dfdxx" in o:
        o["dfdxx"] = o["dfdxx"].reshape(sx, sx).T
    if "K" in o:
        o["K"] = o["K"].reshape(sx, NU).T
    return idx, o


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(1e-300, np.max(np.abs(b))))


def query_times(T):
    ts = [float(T[0]) - 0.1, float(T[-1]) + 0.07]
    ts += [float(v) for v in T]
    ts += [0.5 * (float(T[k]) + float(T[k + 1])) + 1e-4 for k in range(len(T) - 1) if T[k + 1] - T[k] > 1e-6]
    short = [i for i in range(len(T) - 1) if 0 < T[i + 1] - T[i] < 2e-9]
    for i in short:   # inside the short segment, on both sides of its middle
        ts += [float(T[i]) + 0.2e-9, float(T[i]) + 1.3e-9]
    return ts


@pytest.mark.parametrize("fam", list(FAMS))
def test_query_matches_the_restatement(fam):
    sx = FAMS[fam]
    T, ev = plan()
    rng = np.random.default_rng(3)
    Pd, pd, Kd, P, p, K = device_blocks(len(T), sx, rng)
    x = rng.normal(size=sx)
    for tq in query_times(T):
        idx, dev = run(T, ev, Pd, pd, Kd, sx, tq, x)
        r = ref.query(tq, T, ev, P=P, p=p, K=K, x=x)
        assert idx == ref.time_segment(T, tq)[0], tq
        for k in ("dfdxx", "dfdx", "K"):
            assert dev[k].shape == r[k].shape
            assert rel(dev[k], r[k]) <= 1e-15, (k, tq)


@pytest.mark.parametrize("fam", list(FAMS))
def test_segments_the_reference_treats_specially(fam):
    """zero-length and sub-2-weakEpsilon segments snap to an end, t outside the horizon holds an end node, and PreEvent / terminal nodes carry
    the gain of the stage before them"""
    sx = FAMS[fam]
    T, ev = plan()
    n = len(T)
    Pd, pd, Kd, P, p, K = device_blocks(n, sx, np.random.default_rng(4))
    x = np.zeros(sx)
    pre = [k for k in range(1, n) if ev[k] == 1]
    for k in pre:   # on a PreEvent node: alpha = 0 of the segment that ends there -> the node itself, the stage before it
        _, dev = run(T, ev, Pd, pd, Kd, sx, float(T[k]), x)
        assert np.array_equal(dev["K"], K[k - 1]) and np.array_equal(dev["dfdxx"], P[k]), k
    short = [i for i in range(n - 1) if 0 < T[i + 1] - T[i] < 2e-9]
    assert short
    for i in short:
        _, lo = run(T, ev, Pd, pd, Kd, sx, float(T[i]) + 0.2e-9, x)
        _, hi = run(T, ev, Pd, pd, Kd, sx, float(T[i]) + 1.3e-9, x)
        assert np.array_equal(lo["dfdxx"], P[i]) and np.array_equal(hi["dfdxx"], P[i + 1])
    _, before = run(T, ev, Pd, pd, Kd, sx, float(T[0]) - 1.0, x)
    assert np.array_equal(before["dfdxx"], P[0]) and np.array_equal(before["K"], K[0]) and np.array_equal(before["dfdx"], p[0])
    _, past = run(T, ev, Pd, pd, Kd, sx, float(T[-1]) + 1.0, x)   # the terminal node, whose gain is the last stage's
    assert np.array_equal(past["dfdxx"], P[n - 1]) and np.array_equal(past["K"], K[n - 2]) and np.array_equal(past["dfdx"], p[n - 1])


@pytest.mark.parametrize("fam", list(FAMS))
def test_two_node_plans(fam):
    sx = FAMS[fam]
    T, ev = np.array([1.0, 1.04]), np.zeros(2, dtype=np.uint8)
    rng = np.random.default_rng(5)
    Pd, pd, Kd, P, p, K = device_blocks(2, sx, rng)
    x = rng.normal(size=sx)
    for tq in (0.9, 1.0, 1.013, 1.04, 1.2):
        _, dev = run(T, ev, Pd, pd, Kd, sx, tq, x)
        r = ref.query(tq, T, ev, P=P, p=p, K=K, x=x)
        for k in r:
            assert rel(dev[k], r[k]) <= 1e-15, (k, tq)
        assert rel(dev["K"], K[0]) <= 1e-15   # both nodes carry stage 0


def test_outputs_are_independent():
    """an output left out changes none of the others, and the value function alone reads no gains (K = NULL on the device)"""
    T, ev = plan()
    rng = np.random.default_rng(6)
    Pd, pd, Kd, P, p, K = device_blocks(len(T), 58, rng)
    x = rng.normal(size=58)
    tq = 0.4571
    _, full = run(T, ev, Pd, pd, Kd, 58, tq, x)
    _, vf = run(T, ev, Pd, pd, None, 58, tq, x, want=("dfdxx", "dfdx"))
    _, dx = run(T, ev, Pd, pd, None, 58, tq, x, want=("dfdx",))
    _, kk = run(T, ev, None, None, Kd, 58, tq, None, want=("K",))
    assert np.array_equal(vf["dfdxx"], full["dfdxx"]) and np.array_equal(vf["dfdx"], full["dfdx"])
    assert np.array_equal(dx["dfdx"], full["dfdx"]) and np.array_equal(kk["K"], full["K"])


def test_new_entry_points_are_exported():
    assert set(NEW_SYMBOLS) <= set(_l.EXPORTED_SYMBOLS)
    L = _l.lib()
    for name in NEW_SYMBOLS:
        assert hasattr(L, name), name


def test_no_cpu_fallback():
    """without a CUDA device no handle or fleet can be created (B200SQP_ENODEV), so the queries have nothing to run on; called with a null
    handle they fail loudly instead of computing anything"""
    import torch

    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from wb_humanoid_mpc_b200 import model_loader
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    with pytest.raises(_l.B200SqpError) as e:
        B200SqpSolver(model_loader.load_packaged_model())
    assert e.value.code == _l.ENODEV
    L = _l.lib()
    out = np.zeros(NX * NX)
    for name in NEW_SYMBOLS[:4]:
        assert getattr(L, name)(None, C.c_double(0.0), None, _p(out), None, None, None) == _l.EINVAL, name
    assert L.b200sqp_fleet_download_value_function(None, C.c_int(2), _p(out), _p(out), None) == _l.EINVAL
