"""The fleet's device functions on the CPU harness (tests/emu/bld_emu.cu): the stable partition by node count (wb_fleet.cuh) against numpy, and
the builder's warm start from previous solutions of different lengths per instance (wb_builder.cuh, prevLen + slot map) against the host
restatement of SolverBase::preRun (references.py)."""
import numpy as np
import pytest

import bld_emu_lib
from test_emu_builder import compare, make_inputs
from wb_humanoid_mpc_b200 import model_loader, references


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


@pytest.mark.parametrize("B,values,threads", [(1, [40], 1024), (37, [40], 1024), (64, None, 1024), (300, [23, 40, 41, 57], 128), (2500, [30, 31, 33], 1024),
                                              (200, None, 32)])
def test_partition_is_numpys_stable_sort(B, values, threads):
    rng = np.random.default_rng(B + threads)
    nodes = rng.choice(values, B) if values is not None else rng.permutation(np.arange(10, 10 + B))   # None: all counts distinct
    n_bins = int(nodes.max()) + 5
    slot, groups = bld_emu_lib.partition(nodes, n_bins, threads)
    assert np.array_equal(slot, np.argsort(nodes, kind="stable"))
    counts = np.bincount(nodes, minlength=n_bins)
    assert [g[0] for g in groups] == np.flatnonzero(counts).tolist()
    assert [g[2] for g in groups] == counts[counts > 0].tolist()
    assert [g[1] for g in groups] == np.concatenate([[0], np.cumsum(counts[counts > 0])[:-1]]).tolist()


def previous_solutions(model, rng, gaits, starts, x0s, cmds, horizon):
    """made-up previous solutions on each instance's own cold grid (different lengths per instance)"""
    prevs = []
    for b, g in enumerate(gaits):
        h = references.build_instance(model, x0s[b], t0=0.0, horizon=horizon, gait=g, gait_start=(None if g == "stance" else starts[b]), cmd=list(cmds[b]))
        n = len(h["t_nodes"])
        prevs.append(dict(t=np.asarray(h["t_nodes"]), event=np.asarray(h["node_event"]), x=rng.normal(size=(n, 58)), u=rng.normal(size=(n - 1, 35))))
    return prevs


def test_warm_build_with_per_instance_previous_lengths(model):
    rng = np.random.default_rng(11)
    B, horizon = 6, 1.1
    x0s, cmds = make_inputs(model, rng, B)
    gaits = ["stance", "walk", "slow_walk", "walk", "run", "slow_walk"]
    starts = [0.5, -0.13, -0.71, -0.42, -0.05, 0.0]
    prevs = previous_solutions(model, rng, gaits, starts, x0s, cmds, horizon)
    assert len({len(p["t"]) for p in prevs}) > 1
    for t1 in (0.05, 0.3):
        tp = [references.to_primal_solution(p["t"], p["event"], p["x"], p["u"]) for p in prevs]
        x1 = np.array([references.linear_interpolate(t1, p["t"], p["x"]) for p in tp])
        n, dev = bld_emu_lib.warm_build(model, t1, horizon, x1, gaits, starts, cmds, prevs)
        for b in range(B):
            host = references.build_instance(model, x1[b], t0=t1, horizon=horizon, gait=gaits[b], gait_start=(None if gaits[b] == "stance" else starts[b]),
                                             cmd=list(cmds[b]), previous=tp[b])
            assert n[b] == len(host["t_nodes"])
            compare({k: v[None] for k, v in dev[b].items()}, [host])


def test_stateful_warm_build_with_per_instance_previous_lengths(model):
    """the stateful gait schedule: trajectorySpread of previous solutions of different lengths (bldSpreadStrategy / bldSpreadApply with prevLen)
    against the host's GaitSchedule + build_instance(previous = ..., gait_schedule = ...)"""
    rng = np.random.default_rng(17)
    B, horizon, t1 = 6, 1.1, 0.05
    x0s, cmds = make_inputs(model, rng, B)
    gaits = ["stance", "walk", "slow_walk", "walk", "run", "slow_walk"]
    starts = [0.5, -0.13, -0.71, -0.42, -0.05, 0.0]
    schedules, prevs, tp = [], [], []
    for b, g in enumerate(gaits):   # the host's cold build at t = 0 (test_gpu_gait_schedule.HostLoop)
        gs = references.GaitSchedule()
        if g != "stance":
            g_ = model["gaits"][g]
            gs.insert_template([references.MODE_NAMES[m] for m in g_["modeSequence"]], g_["switchingTimes"], starts[b], 2 * horizon)
        h = references.build_instance(model, x0s[b], t0=0.0, horizon=horizon, cmd=list(cmds[b]), gait_schedule=gs)
        n = len(h["t_nodes"])
        p = dict(t=np.asarray(h["t_nodes"]), event=np.asarray(h["node_event"]), x=rng.normal(size=(n, 58)), u=rng.normal(size=(n - 1, 35)))
        prevs.append(p)
        tp.append(references.to_primal_solution(p["t"], p["event"], p["x"], p["u"], mode_schedule=h["mode_schedule"]))
        schedules.append(gs)
    assert len({len(p["t"]) for p in prevs}) > 1
    x1 = np.array([references.linear_interpolate(t1, p["t"], p["x"]) for p in tp])
    n, dev = bld_emu_lib.warm_build(model, t1, horizon, x1, gaits, starts, cmds, prevs, stateful=True, t_prev=0.0)
    for b in range(B):
        host = references.build_instance(model, x1[b], t0=t1, horizon=horizon, cmd=list(cmds[b]), previous=tp[b], gait_schedule=schedules[b])
        assert n[b] == len(host["t_nodes"])
        compare({k: v[None] for k, v in dev[b].items()}, [host])


def test_uniform_path_is_unchanged(model):
    """null prevLen and slot map: bitwise the builder of a plain handle"""
    rng = np.random.default_rng(3)
    B, horizon = 3, 1.1
    x0s, cmds = make_inputs(model, rng, B)
    prevs = previous_solutions(model, rng, ["walk"] * B, [0.0] * B, x0s, cmds, horizon)
    n, dev = bld_emu_lib.warm_build(model, 0.2, horizon, x0s, ["walk"] * B, [0.0] * B, cmds, prevs, per_instance=False)
    ref = bld_emu_lib.build_instances(model, 0.2, horizon, x0s, ["walk"] * B, [0.0] * B, cmds,
                                  previous=dict(t=[p["t"] for p in prevs], event=[p["event"] for p in prevs], x=[p["x"] for p in prevs], u=[p["u"] for p in prevs]))
    for b in range(B):
        for k in dev[b]:
            assert np.array_equal(dev[b][k], ref[k][b]), k
    # and the per-instance path with equal lengths gives the same bits
    n2, dev2 = bld_emu_lib.warm_build(model, 0.2, horizon, x0s, ["walk"] * B, [0.0] * B, cmds, prevs)
    assert np.array_equal(n, n2)
    for b in range(B):
        for k in dev[b]:
            assert np.array_equal(dev[b][k], dev2[b][k]), k
