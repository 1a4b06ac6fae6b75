"""The C-ABI library loads and exports exactly what include/b200sqp.h declares; no compute calls (no GPU here)."""
import ctypes as C
import re
from pathlib import Path

import pytest

from wb_humanoid_mpc_b200 import abi, lib

ROOT = Path(__file__).resolve().parents[1]


def header_symbols():
    text = (ROOT / "include" / "b200sqp.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200sqp_[a-z_0-9]+)\s*\(", text)))


def test_header_and_loader_agree():
    assert header_symbols() == sorted(lib.EXPORTED_SYMBOLS)


def test_return_codes_match_header():
    text = (ROOT / "include" / "b200sqp.h").read_text()
    codes = {m[0]: int(m[1]) for m in re.findall(r"#define B200SQP_(E[A-Z]+)\s+(-?\d+)", text)}
    assert codes == {name: getattr(lib, name) for name in ("EINVAL", "ENODEV", "ENOMEM", "EQP", "ESTATE")}


def test_library_exports_every_declared_symbol():
    L = lib.lib()
    for name in header_symbols():
        assert hasattr(L, name), f"{name} declared in include/b200sqp.h but not exported by libb200sqp.so"
    assert b"sm_90a" in L.b200sqp_version()


def test_struct_sizes_match_header():
    """ctypes mirrors vs the C compiler's view of the structs (compiled probe)."""
    import subprocess
    import tempfile

    src = '#include "b200sqp.h"\n#include <stdio.h>\nint main(){printf("%zu %zu %zu\\n", sizeof(b200sqp_model_desc), sizeof(b200sqp_settings), sizeof(b200sqp_iter_log));}\n'
    with tempfile.TemporaryDirectory() as td:
        p = Path(td) / "probe.c"
        p.write_text(src)
        exe = Path(td) / "probe"
        subprocess.run(["gcc", "-I", str(ROOT / "include"), str(p), "-o", str(exe)], check=True)
        sizes = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [C.sizeof(abi.ModelDesc), C.sizeof(abi.Settings), C.sizeof(abi.IterLog)]


def test_no_cpu_fallback():
    """without a CUDA device every computing entry point must fail loudly (B200SQP_ENODEV), never fall back to the CPU"""
    import torch

    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from wb_humanoid_mpc_b200 import model_loader
    from wb_humanoid_mpc_b200.qp import BatchedQp
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    with pytest.raises(lib.B200SqpError) as e1:
        BatchedQp(1, 4, 3, 2)
    assert e1.value.code == -2
    with pytest.raises(lib.B200SqpError) as e2:
        B200SqpSolver(model_loader.load_packaged_model())
    assert e2.value.code == -2


def test_product_does_not_import_the_oracle():
    """nothing under wb_humanoid_mpc_b200/ may reference oracle/ or the CPU dev harness"""
    for p in (ROOT / "wb_humanoid_mpc_b200").rglob("*"):
        if p.suffix in (".py", ".cu", ".cuh", ".inc", ".h"):
            t = p.read_text()
            assert "oracle_lib" not in t and "liboracle" not in t and "libwbemu" not in t and "orc_" not in t, p


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: no source of the product package may import, include, link or dlopen it (only tests/, smoke() and
    bench.py's CPU legs do)"""
    import re
    from pathlib import Path

    root = Path(__file__).resolve().parents[1]
    pat = re.compile(r"(import\s+oracle_lib|from\s+oracle_lib|liboracle|#include\s+[\"<][^\"<>]*oracle/|\borc_[a-z_]+\s*\()")
    bad = []
    for f in (root / "wb_humanoid_mpc_b200").rglob("*"):
        if f.suffix in {".py", ".cpp", ".hpp", ".cu", ".cuh", ".inc", ".h"}:
            for n, line in enumerate(f.read_text(errors="ignore").splitlines(), 1):
                if pat.search(line):
                    bad.append(f"{f.relative_to(root)}:{n}: {line.strip()}")
    for f in (root / "include").glob("*.h"):
        if pat.search(f.read_text()):
            bad.append(str(f))
    assert not bad, "\n".join(bad)
    # bench.py: the oracle only inside the CPU-baseline / reference legs
    src = (root / "bench.py").read_text()
    assert src.count("import oracle_lib") <= 2 and "def oracle_batch_solve" in src
