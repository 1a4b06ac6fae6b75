"""include/ocs2_sqp/B200SqpSolver.h -- the ocs2::SolverBase drop-in a wb_humanoid_mpc workspace puts behind SqpMpc (SURVEY.md section 8b, INTEGRATION.md) --
compiled with g++ against the stand-in ocs2 headers of tests/stubs/ and driven like SqpMpc::calculateController drives ocs2::SqpSolver
(tests/stubs/shim_test.cpp).  CPU: it compiles, links against libb200sqp.so and refuses to run without a device (no CPU fallback).  GPU: two MPC
cycles (cold, then warm start from its own PrimalSolution); the first solution equals the batched C++ host layer's on the same instance."""
import subprocess
from pathlib import Path

import pytest

from wb_humanoid_mpc_b200 import lib

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def shim_exe(tmp_path_factory):
    """tests/stubs/shim_test.cpp built once per module in a temporary directory, so that the suite also runs from a read-only tree"""
    lib.lib()   # make sure libb200sqp.so exists
    exe = tmp_path_factory.mktemp("shim") / "shim_test"
    pkg = ROOT / "wb_humanoid_mpc_b200"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", f"-I{ROOT / 'include'}", f"-I{ROOT / 'tests' / 'stubs'}", "-o", str(exe), str(ROOT / "tests" / "stubs" / "shim_test.cpp"),
                    f"-L{pkg}", "-lb200sqp", "-pthread", f"-Wl,-rpath,{pkg}"], check=True, cwd=ROOT)
    return exe


def run_shim(exe):
    return subprocess.run([str(exe), str(ROOT / "wb_humanoid_mpc_b200" / "data" / "g1_wb_model.txt")], capture_output=True, text=True, cwd=ROOT, timeout=300)


def test_shim_compiles_against_stub_ocs2_and_fails_loudly_without_a_device(shim_exe):
    import torch

    out = run_shim(shim_exe)
    if torch.cuda.is_available():
        assert out.returncode == 0, out.stdout + out.stderr
    else:
        assert out.returncode == 3 and "no CUDA device" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_shim_two_mpc_cycles_match_the_host_layer(shim_exe):
    out = run_shim(shim_exe)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM_OK" in out.stdout
