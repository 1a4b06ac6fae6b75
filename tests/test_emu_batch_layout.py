"""The batch layout of a handle (wb_batch.cuh) on the CPU harness (tests/emu/bld_emu.cu): which arrays set_batch allocates under which settings
and at what size, the group views of a fleet (groupView) inside their allocations and apart from each other, and the slot helper of the slot
kernels (fleetSlot, wb_fleet.cuh) on the rows of those views."""
import itertools

import numpy as np
import pytest

import bld_emu_lib

NX, NU, NUT_MAX = 58, 35, 23
MAX_ITER, RAW_PER = 3, 1234   # the widths of log and raw (settings.sqp_iteration, the raw block's doubles)
# set_batch's arrays: row kind and elements per row (None: a record size of wb_solver.cuh)
ARRAYS = {
    "x0": ("instance", NX), "x": ("node", NX), "u": ("stage", NU), "xInit": ("node", NX), "uInit": ("stage", NU), "t": ("node", 1),
    "swing": ("node", 6), "impact": ("node", 2), "arm": ("node", 1), "xref": ("node", NX), "event": ("node", 1), "contact": ("node", 2),
    "qp.A": ("stage", NX * NX), "qp.Bm": ("stage", NX * NUT_MAX), "qp.b": ("stage", NX), "qp.Q": ("node", NX * NX), "qp.S": ("stage", NUT_MAX * NX),
    "qp.R": ("stage", NUT_MAX * NUT_MAX), "qp.q": ("node", NX), "qp.r": ("stage", NUT_MAX), "qp.dx0": ("instance", NX), "qp.nu": ("stage", 1),
    "qp.K": ("stage", NUT_MAX * NX), "qp.kff": ("stage", NUT_MAX), "qp.p": ("node", NX), "qp.P": ("node", NX * NX), "qp.dx": ("node", NX),
    "qp.du": ("stage", NUT_MAX), "qp.status": ("instance", 1), "Pu": ("stage", NU * NUT_MAX), "Px": ("stage", NU * NX), "u0p": ("stage", NU),
    "du": ("stage", NU), "Kre": ("stage", NU * NX), "perfNode": ("node", 4), "lsNode": ("node", 4), "inst": ("instance", 16), "flags": ("instance", 8),
    "pending": ("handle", 1), "log": ("instance", MAX_ITER), "mid": ("stage", None), "luRec": ("stage", None), "luPerm": ("stage", 52),
    "gstats": ("handle", 32 * 4 + 8), "raw": ("stage", RAW_PER),
}
# whole-body / centroidal, create_value_function, use_feedback_policy, raw capture
CONFIGS = [dict(cen=c, value_function=v, feedback=f, raw=r) for c, v, f, r in itertools.product((False, True), repeat=4)]
IDS = ["{}{}{}{}".format("cen" if c["cen"] else "wb", "-vf" * c["value_function"], "-fb" * c["feedback"], "-raw" * c["raw"]) for c in CONFIGS]
# three groups of different node counts below the capacity, in slot order
B, CAP = 9, 30
GROUPS = [(12, 0, 2), (17, 2, 4), (25, 6, 3)]


def rows(kind, count, nodes):
    return {"instance": count, "node": count * nodes, "stage": count * (nodes - 1), "handle": 1}[kind]


def layout(config):
    return bld_emu_lib.batch_layout(**config, max_iter=MAX_ITER, raw_per=RAW_PER)


@pytest.mark.parametrize("config", CONFIGS, ids=IDS)
def test_the_table_holds_set_batchs_arrays_under_its_conditions(config):
    entries = layout(config)
    names = [e[0] for e in entries]
    assert len(set(names)) == len(names)
    conditional = {"qp.P": config["value_function"], "Kre": config["feedback"], "mid": not config["cen"], "luRec": not config["cen"],
                   "luPerm": not config["cen"], "raw": config["raw"]}
    assert set(names) == {k for k in ARRAYS if conditional.get(k, True)}
    for name, kind, width, _ in entries:
        assert kind == ARRAYS[name][0], name
        assert ARRAYS[name][1] in (None, width), name
    assert {e[0] for e in entries if e[3]} == ({"x0", "x", "xref"} if config["cen"] else set())   # the padded state rows


@pytest.mark.parametrize("config", CONFIGS, ids=IDS)
def test_group_views_lie_inside_their_allocations_and_apart(config):
    entries = layout(config)
    nbytes, off = bld_emu_lib.group_views(**config, max_iter=MAX_ITER, raw_per=RAW_PER, B=B, cap=CAP, groups=GROUPS)
    assert len(nbytes) == len(entries)
    for e, (name, kind, width, _) in enumerate(entries):
        esz = nbytes[e] // (rows(kind, B, CAP) * width)
        assert nbytes[e] == rows(kind, B, CAP) * width * esz, name
        if kind == "handle":   # handle-wide: every view keeps the base's array, except the line-search counter it is given (null here)
            assert (off[:, e] == (-1 if name == "pending" else 0)).all(), name
            continue
        spans = sorted((off[g, e], off[g, e] + rows(kind, count, n) * width * esz) for g, (n, first, count) in enumerate(GROUPS))
        assert spans[0][0] >= 0 and spans[-1][1] <= nbytes[e], name
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), name


@pytest.mark.parametrize("config", CONFIGS, ids=IDS)
def test_one_group_of_the_whole_batch_is_the_base(config):
    entries = layout(config)
    nbytes, off = bld_emu_lib.group_views(**config, max_iter=MAX_ITER, raw_per=RAW_PER, B=B, cap=CAP, groups=[(CAP, 0, B)])
    for e, (name, kind, _, _) in enumerate(entries):
        assert off[0, e] == (-1 if name == "pending" else 0), name


def test_the_slot_helper_rows_are_the_group_views_rows():
    config = CONFIGS[0]
    entries = [e[0] for e in layout(config)]
    _, off = bld_emu_lib.group_views(**config, max_iter=MAX_ITER, raw_per=RAW_PER, B=B, cap=CAP, groups=GROUPS)
    x, u = entries.index("x"), entries.index("u")
    sl = bld_emu_lib.fleet_slots(GROUPS, B, CAP)
    for g, (n, first, count) in enumerate(GROUPS):
        for s in range(first, first + count):
            assert (sl["n"][s], sl["first"][s], sl["count"][s]) == (n, first, count)
            assert sl["node"][s] == off[g, x] // (NX * 8) + (s - first) * n
            assert sl["stage"][s] == off[g, u] // (NU * 8) + (s - first) * (n - 1)
    plain = bld_emu_lib.fleet_slots(None, B, CAP)   # a plain handle: one group of the batch at its node count
    s = np.arange(B)
    assert (plain["n"] == CAP).all() and (plain["first"] == 0).all() and (plain["count"] == B).all()
    assert np.array_equal(plain["node"], s * CAP) and np.array_equal(plain["stage"], s * (CAP - 1))
