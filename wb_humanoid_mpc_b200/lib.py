"""Loader/build helper for the C-ABI shared library (wb_humanoid_mpc_b200/libb200sqp.so).

The library is built in-tree with nvcc for sm_90a (H100) (see `build`).  There is no CPU fallback: if the library is
missing, or no CUDA device is present, every computing entry point fails loudly (B200SQP_ENODEV).
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
SO = Path(os.environ["B200SQP_LIB"]) if os.environ.get("B200SQP_LIB") else PKG / "libb200sqp.so"  # override: development builds only
INCLUDE = PKG.parent / "include"

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
              "-DB200SQP_WITH_WB"]

dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)
u8p = C.POINTER(C.c_uint8)

# the return codes of include/b200sqp.h (B200SQP_E*; tests/test_abi.py checks them against the header)
EINVAL, ENODEV, ENOMEM, EQP, ESTATE = -1, -2, -3, -4, -5


class B200SqpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200sqp error {code}: {msg}")
        self.code = code


def sources():
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.inc")) + [INCLUDE / "b200sqp.h"])


def needs_build() -> bool:
    if not SO.exists():
        return True
    if os.environ.get("B200SQP_LIB"):
        return False   # a development build made by hand (own -D flags): never rebuilt from here
    t = SO.stat().st_mtime
    return any(s.stat().st_mtime > t for s in sources())


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source for sm_90a into libb200sqp.so (cross-compiles without a GPU)."""
    if not force and not needs_build():
        return SO
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    flags = list(NVCC_FLAGS) + os.environ.get("B200SQP_NVCC_EXTRA", "").split()  # extra flags: development builds only
    if not (CSRC / "wb_solver.cuh").exists():
        flags.remove("-DB200SQP_WITH_WB")
    cmd = [nvcc, *flags, "-o", str(SO), str(CSRC / "b200sqp.cu")]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return SO


_lib = None


def lib() -> C.CDLL:
    """dlopen the C-ABI library; builds it first when sources are newer and nvcc is available."""
    global _lib
    if _lib is not None:
        return _lib
    if needs_build():
        if SO.exists() and not (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")):
            pass  # stale but usable (GPU box without toolchain changes)
        else:
            build()
    if not SO.exists():
        raise B200SqpError(-2, f"{SO} is missing and could not be built; there is no CPU fallback")
    L = C.CDLL(str(SO))
    L.b200sqp_last_error.restype = C.c_char_p
    L.b200sqp_version.restype = C.c_char_p
    for name in EXPORTED_SYMBOLS:
        try:
            fn = getattr(L, name)
        except AttributeError:  # reported by tests/test_abi.py; do not mask the symbols that do exist
            continue
        if name not in ("b200sqp_last_error", "b200sqp_version", "b200sqp_qp_destroy", "b200sqp_destroy", "b200sqp_default_settings",
                        "b200sqp_default_rollout_settings", "b200sqp_host_alloc", "b200sqp_host_free", "b200sqp_fleet_destroy"):
            fn.restype = C.c_int
    if hasattr(L, "b200sqp_host_alloc"):
        L.b200sqp_host_alloc.restype = C.c_void_p
        L.b200sqp_host_alloc.argtypes = [C.c_size_t]
        L.b200sqp_host_free.restype = None
        L.b200sqp_host_free.argtypes = [C.c_void_p]
    for name in ("b200sqp_qp_destroy", "b200sqp_destroy", "b200sqp_default_settings", "b200sqp_default_rollout_settings", "b200sqp_fleet_destroy"):
        if hasattr(L, name):
            getattr(L, name).restype = None
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise B200SqpError(rc, lib().b200sqp_last_error().decode())


# every symbol include/b200sqp.h declares (tests/test_abi.py cross-checks this list against the header)
EXPORTED_SYMBOLS = [
    "b200sqp_last_error",
    "b200sqp_version",
    "b200sqp_qp_create",
    "b200sqp_qp_destroy",
    "b200sqp_qp_upload",
    "b200sqp_qp_solve",
    "b200sqp_qp_download",
    "b200sqp_qp_last_ms",
    "b200sqp_default_settings",
    "b200sqp_create",
    "b200sqp_destroy",
    "b200sqp_set_batch",
    "b200sqp_upload_instances",
    "b200sqp_host_alloc",
    "b200sqp_host_free",
    "b200sqp_reset",
    "b200sqp_solve",
    "b200sqp_wait",
    "b200sqp_own_stream",
    "b200sqp_set_builder",
    "b200sqp_build_instances",
    "b200sqp_download_instances",
    "b200sqp_set_gait_schedule",
    "b200sqp_download_mode_schedule",
    "b200sqp_set_motion_manager",
    "b200sqp_download_motion_state",
    "b200sqp_cen_set_gait_schedule",
    "b200sqp_set_joint_torque_cost",
    "b200sqp_cen_set_motion_manager",
    "b200sqp_default_rollout_settings",
    "b200sqp_rollout_policy",
    "b200sqp_cen_rollout_policy",
    "b200sqp_joint_actions",
    "b200sqp_set_comm",
    "b200sqp_global_stats",
    "b200sqp_global_ladder",
    "b200sqp_line_search_trials",
    "b200sqp_download",
    "b200sqp_download_value_function",
    "b200sqp_centroidal_flow_map",
    "b200sqp_cen_create",
    "b200sqp_joint_torques",
    "b200sqp_download_stage_blocks",
    "b200sqp_stage_doubles",
    "b200sqp_get_stage_times",
    "b200sqp_get_launch_count",
    "b200sqp_fleet_create",
    "b200sqp_fleet_destroy",
    "b200sqp_fleet_build_instances",
    "b200sqp_fleet_solve",
    "b200sqp_fleet_wait",
    "b200sqp_fleet_rollout_policy",
    "b200sqp_fleet_joint_actions",
    "b200sqp_fleet_download",
    "b200sqp_fleet_download_instances",
    "b200sqp_fleet_download_mode_schedule",
    "b200sqp_fleet_get_stage_times",
    "b200sqp_fleet_download_motion_state",
    "b200sqp_set_reset_states",
    "b200sqp_set_auto_reset",
    "b200sqp_request_resets",
    "b200sqp_download_episodes",
    "b200sqp_fleet_set_reset_states",
    "b200sqp_fleet_request_resets",
    "b200sqp_fleet_download_episodes",
    "b200sqp_set_pose_commands",
    "b200sqp_command_poses",
    "b200sqp_clear_poses",
    "b200sqp_download_pose_targets",
    "b200sqp_fleet_command_poses",
    "b200sqp_fleet_clear_poses",
    "b200sqp_fleet_download_pose_targets",
    "b200sqp_build_instances_dev",
    "b200sqp_fleet_build_instances_dev",
    "b200sqp_joint_actions_dev",
    "b200sqp_fleet_joint_actions_dev",
    "b200sqp_download_dev",
    "b200sqp_fleet_download_dev",
    "b200sqp_mrt_query",
    "b200sqp_fleet_mrt_query",
    "b200sqp_mrt_query_dev",
    "b200sqp_fleet_mrt_query_dev",
    "b200sqp_fleet_download_value_function",
    "b200sqp_default_gains",
    "b200sqp_set_gains",
    "b200sqp_download_gains",
    "b200sqp_set_gains_dev",
    "b200sqp_fleet_set_gains",
    "b200sqp_fleet_download_gains",
    "b200sqp_fleet_set_gains_dev",
    "b200sqp_default_robot_params",
    "b200sqp_set_robot_params",
    "b200sqp_download_robot_params",
    "b200sqp_set_robot_params_dev",
    "b200sqp_fleet_set_robot_params",
    "b200sqp_fleet_download_robot_params",
    "b200sqp_fleet_set_robot_params_dev",
]
