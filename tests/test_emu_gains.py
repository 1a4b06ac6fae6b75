"""Per-instance gains without a GPU: the row functions of gains_apply_kernel (wb_gains.cuh) executed on the host (tests/emu).  The model they
make from a gain set is byte for byte the model the handle's constructor makes from a model description carrying that gain set, on both
families, and every invalid field is rejected with its status.  The launches are checked by tests/test_gpu_gains.py."""
import copy
import ctypes as C

import numpy as np
import pytest

from emu_build import build
from wb_humanoid_mpc_b200 import abi, model_loader

FAMILIES = ["g1_wb", "g1_centroidal"]


def is_cen(model) -> bool:
    return model.get("kind") == "centroidal"


def model_gains(model) -> dict:
    """the gain record of a model dictionary, every term active (what b200sqp_default_gains returns for a handle made from it)"""
    g = {k: np.zeros(abi.GAINS_DTYPE[k].shape) for k in abi.GAIN_FIELDS}
    for k, src in (("Q_diag", "Q_diag"), ("R_diag", "R_diag"), ("Qf_diag", "Qf_diag"), ("foot_cost_w", "foot_cost_weights")):
        g[k][: len(model[src])] = model[src]
    if is_cen(model):
        g["torso_w"][:12] = model["task_space_cost"]["weights"]
    g["jlim_mu"], g["jlim_delta"] = model["joint_limits"]["mu"], model["joint_limits"]["delta"]
    c = model["collision"]
    g["coll_mu"], g["coll_delta"], g["coll_r_foot"], g["coll_r_knee"] = c["mu"], c["delta"], c["r_foot"], c["r_knee"]
    g["fric_mu"], g["fric_delta"] = model["friction"]["mu"], model["friction"]["delta"]
    g["momxy_mu"], g["momxy_delta"] = model["moment_xy"]["mu"], model["moment_xy"]["delta"]
    for k in abi.GAIN_FIELDS:
        if k.endswith("_active"):
            g[k] = 1
    return g


def random_gains(model, rng, inactive=()) -> dict:
    """a seeded gain set around the model's: Q, R, Q_final, foot and task-space weights scaled by U[0.5, 2] per entry, penalty mu and delta
    by U[0.5, 2], the radii by U[0.8, 1.2]; the terms named in `inactive` switched off"""
    g = model_gains(model)
    for k in ("Q_diag", "R_diag", "Qf_diag", "foot_cost_w", "torso_w"):
        g[k] = g[k] * rng.uniform(0.5, 2.0, g[k].shape)
    for k in ("jlim_mu", "jlim_delta", "coll_mu", "coll_delta", "fric_mu", "fric_delta", "momxy_mu", "momxy_delta"):
        g[k] = g[k] * rng.uniform(0.5, 2.0)
    for k in ("coll_r_foot", "coll_r_knee"):
        g[k] = g[k] * rng.uniform(0.8, 1.2)
    for k in inactive:
        g[k] = 0
    return g


def model_with_gains(model, g) -> dict:
    """the model dictionary whose description carries gain set g: an inactive term has zero weights (costs) or a zero mu (penalties)"""
    m = copy.deepcopy(model)
    on = lambda k: bool(g[k])
    nx, nu = len(model["Q_diag"]), len(model["R_diag"])
    m["Q_diag"] = list(g["Q_diag"][:nx])
    m["R_diag"] = list(g["R_diag"][:nu])
    m["Qf_diag"] = list(g["Qf_diag"][:nx] if on("final_cost_active") else np.zeros(nx))
    nf = len(model["foot_cost_weights"])
    m["foot_cost_weights"] = list(g["foot_cost_w"][:nf] if on("foot_cost_active") else np.zeros(nf))
    if is_cen(model):
        m["task_space_cost"]["weights"] = list(g["torso_w"][:12] if on("torso_cost_active") else np.zeros(12))
    m["joint_limits"].update(mu=float(g["jlim_mu"]) if on("joint_limits_active") else 0.0, delta=float(g["jlim_delta"]))
    m["collision"].update(mu=float(g["coll_mu"]) if on("foot_collision_active") else 0.0, delta=float(g["coll_delta"]),
                          r_foot=float(g["coll_r_foot"]), r_knee=float(g["coll_r_knee"]))
    m["friction"].update(mu=float(g["fric_mu"]) if on("friction_cone_active") else 0.0, delta=float(g["fric_delta"]))
    m["moment_xy"].update(mu=float(g["momxy_mu"]) if on("contact_moment_active") else 0.0, delta=float(g["momxy_delta"]))
    return m


def record(g) -> abi.Gains:
    return abi.Gains.from_buffer_copy(abi.pack_gains(g, 1).tobytes())


_lib = None


def device_model(model, g=None) -> tuple[int, bytes]:
    """(row status, device-model bytes) of the gains row (tests/emu/gains_emu.cu) on the model of `model`; g = None: that model itself"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build("gains_emu.cu", "libgainsemu.so")))
    cd = abi.cen_desc(model) if is_cen(model) else None
    out, n = (C.c_uint8 * 32768)(), C.c_int64(0)
    rc = _lib.emu_gains_model(C.byref(abi.model_desc(model)), None if cd is None else C.byref(cd), None if g is None else C.byref(record(g)), out,
                              C.byref(n))
    return rc, bytes(out)[: n.value]


@pytest.fixture(scope="module", params=FAMILIES)
def model(request):
    return model_loader.load_packaged_model(request.param)


ACTIVE = [k for k in abi.GAIN_FIELDS if k.endswith("_active")]


@pytest.mark.parametrize("seed", range(6))
def test_applied_model_is_the_model_of_the_modified_description(model, seed):
    rng = np.random.default_rng(seed)
    inactive = [k for k in ACTIVE if rng.uniform() < 0.3] if seed else []
    g = random_gains(model, rng, inactive)
    st, got = device_model(model, g)
    assert st == 0
    rc, want = device_model(model_with_gains(model, g))
    assert rc == 0 and len(got) == len(want)
    assert got == want


def test_default_gains_reproduce_the_model(model):
    st, got = device_model(model, model_gains(model))
    assert st == 0
    assert got == device_model(model)[1]


def test_inactive_terms_zero_their_weights_or_mu(model):
    g = random_gains(model, np.random.default_rng(11), ACTIVE)
    st, got = device_model(model, g)
    assert st == 0
    zero = model_gains(model)
    for k in ("Qf_diag", "foot_cost_w", "torso_w", "jlim_mu", "coll_mu", "fric_mu", "momxy_mu"):
        zero[k] = np.zeros_like(np.asarray(zero[k], float))
    for k in ("Q_diag", "R_diag", "jlim_delta", "coll_delta", "coll_r_foot", "coll_r_knee", "fric_delta", "momxy_delta"):
        zero[k] = g[k]
    assert got == device_model(model_with_gains(model, zero))[1]


# (field, entry or None, value, expected status): 1 = not finite, 2 = out of range
REJECTIONS = [
    ("Q_diag", 3, -1.0, 2), ("Q_diag", 0, np.nan, 1), ("Q_diag", 5, np.inf, 1),
    ("Qf_diag", 1, -1e-3, 2), ("Qf_diag", 2, np.nan, 1), ("Qf_diag", 4, -np.inf, 1),
    ("R_diag", 0, 0.0, 2), ("R_diag", 7, -2.0, 2), ("R_diag", 1, np.nan, 1), ("R_diag", 2, np.inf, 1),
    ("foot_cost_w", 2, -1.0, 2), ("foot_cost_w", 0, np.nan, 1), ("foot_cost_w", 11, np.inf, 1),
    ("jlim_mu", None, -0.1, 2), ("jlim_mu", None, np.nan, 1), ("jlim_delta", None, 0.0, 2), ("jlim_delta", None, np.inf, 1),
    ("coll_mu", None, -1.0, 2), ("coll_delta", None, 0.0, 2), ("coll_delta", None, -1.0, 2), ("coll_r_foot", None, -0.01, 2),
    ("coll_r_knee", None, np.nan, 1), ("coll_r_foot", None, np.inf, 1),
    ("fric_mu", None, -1.0, 2), ("fric_delta", None, 0.0, 2), ("fric_delta", None, np.nan, 1),
    ("momxy_mu", None, np.inf, 1), ("momxy_delta", None, 0.0, 2), ("momxy_delta", None, -0.5, 2),
] + [(k, None, 2, 2) for k in ACTIVE] + [(k, None, -1, 2) for k in ACTIVE[:2]]


@pytest.mark.parametrize("field,entry,value,status", REJECTIONS, ids=[f"{f}-{e}-{v}" for f, e, v, _ in REJECTIONS])
def test_validation_table(model, field, entry, value, status):
    g = model_gains(model)
    if entry is None:
        g[field] = value
    else:
        g[field][entry] = value
    assert device_model(model, g)[0] == status


def test_validation_reads_only_the_used_entries(model):
    cen = is_cen(model)
    g = model_gains(model)
    nx, nu = (35, 35) if cen else (58, 35)
    g["Q_diag"][nx:] = np.nan
    g["Qf_diag"][nx:] = -1.0
    g["R_diag"][nu:] = 0.0
    g["foot_cost_w"][12 if cen else 18:] = np.nan
    if not cen:
        g["torso_w"][:] = -1.0   # ignored on whole-body handles
    assert device_model(model, g)[0] == 0
    if cen:
        g["torso_w"][4] = -1.0
        assert device_model(model, g)[0] == 2
        g["torso_w"][4] = np.nan
        assert device_model(model, g)[0] == 1


def test_pack_roundtrip():
    rng = np.random.default_rng(3)
    g = random_gains(model_loader.load_packaged_model("g1_wb"), rng, ["torso_cost_active"])
    rows = abi.pack_gains({k: np.stack([np.asarray(v)] * 3) for k, v in g.items()})
    assert rows.shape == (3, abi.GAINS_BYTES) and abi.GAINS_BYTES == 1760
    back = abi.unpack_gains(rows)
    for k in abi.GAIN_FIELDS:
        np.testing.assert_array_equal(back[k][1], g[k])
