"""CPU: the C-ABI library builds, loads and exports every symbol include/cgd_b200.h declares; the Python op tables
match the header; product entry points fail loudly without CUDA (no fallback)."""
import ctypes
import os
import re

import pytest
import torch as th

import __graft_entry__ as ge
from clip_guided_diffusion_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "cgd_b200.h")).read()


@pytest.fixture(scope="module")
def lib():
    ge.build()
    return _lib.load()


def test_header_symbols_exported_abi_v3(lib):
    declared = set(re.findall(r"^(?:int|const char\*)\s+(cgd_\w+)\s*\(", HEADER, flags=re.M))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.cgd_abi_version() == 3


def test_op_tables_match_header():
    ops = dict((k, int(v)) for k, v in re.findall(r"CGD_OP_(\w+) = (\d+)", HEADER))
    assert ops == _lib.OP
    sc = dict((k, int(v)) for k, v in re.findall(r"CGD_SC_(\w+) = (\d+)", HEADER))
    sc.pop("_COUNT", None)
    exp = {k: v for k, v in _lib.SC.items() if k != "COUNT"}
    assert sc == exp
    assert ctypes.sizeof(_lib.CgdOp) == 8 + 24 * 8 + 8 * 4 + 12 * 8


def test_plan_create_validates(lib):
    bad = (_lib.CgdOp * 1)()
    bad[0].code = 999
    h = ctypes.c_void_p()
    assert lib.cgd_plan_create(bad, 1, ctypes.byref(h)) != 0
    assert b"unknown code" in lib.cgd_last_error()
    bad[0].code = 31  # retired (batched-GEMM attention softmax): rejected when the plan is built, not when it runs
    assert lib.cgd_plan_create(bad, 1, ctypes.byref(h)) != 0
    assert b"unknown code" in lib.cgd_last_error()
    bad[0].code = _lib.OP["CONV"]
    bad[0].i[20] = 8  # reserved operand (was the batched-B mode)
    assert lib.cgd_plan_create(bad, 1, ctypes.byref(h)) != 0
    assert b"reserved" in lib.cgd_last_error()
    bad[0].i[20] = 0  # all-zero conv: rejected by argument validation before any CUDA call
    assert lib.cgd_plan_create(bad, 1, ctypes.byref(h)) != 0
    assert b"conv" in lib.cgd_last_error()


@pytest.mark.skipif(th.cuda.is_available(), reason="CPU-only check")
def test_no_cpu_fallback():
    from clip_guided_diffusion_b200.plan import Plan
    p = Plan()
    b = p.new(16, "f")
    p.emit("QGELU_FWD", i=[16], p=[(b, 0), (b, 0)])
    p.finalize("cpu")
    with pytest.raises(_lib.CgdError):
        p.run()


def test_header_is_plain_c_abi_v3(tmp_path):
    """include/cgd_b200.h is the FFI contract: it must compile as C (no C++ or torch types) and link against the built library"""
    import shutil, subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "probe.c"
    src.write_text('#include "cgd_b200.h"\n#include <stdio.h>\n'
                   'int main(void) { CgdOp op; (void)op; printf("%d %d\\n", cgd_abi_version(), (int)sizeof(CgdOp)); return 0; }\n')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(_lib.LIB_PATH)
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe), "-L", libdir,
                        "-l:libcgd_b200.so", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.split() == ["3", str(8 + 24 * 8 + 8 * 4 + 12 * 8)], out.stdout + out.stderr


def test_product_path_never_imports_the_oracle():
    """`oracle/` is test infrastructure: nothing under the package may import it, and bench.py only inside its CPU / PyTorch-CUDA
    baseline legs (`oracle_cpu_setup`, `torch_cuda_baseline`) -- never in the engine construction or the timed loops of the own arm"""
    import ast
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def oracle_imports(path):
        tree = ast.parse(open(path).read())
        hits = []
        for fn in ast.walk(tree):
            if isinstance(fn, (ast.FunctionDef, ast.Module)):
                for node in (fn.body if isinstance(fn, ast.FunctionDef) else [n for n in fn.body if not isinstance(n, (ast.FunctionDef, ast.ClassDef))]):
                    for sub in ast.walk(node):
                        mod = sub.module if isinstance(sub, ast.ImportFrom) else (sub.names[0].name if isinstance(sub, ast.Import) else None)
                        if mod and (mod == "oracle" or mod.startswith("oracle.")):
                            hits.append(getattr(fn, "name", "<module>"))
        return set(hits)

    pkg = os.path.join(root, "clip_guided_diffusion_b200")
    for f in sorted(os.listdir(pkg)):
        if f.endswith(".py"):
            assert not oracle_imports(os.path.join(pkg, f)), f"{f} imports the oracle"
    assert oracle_imports(os.path.join(root, "bench.py")) == {"oracle_cpu_setup", "torch_cuda_baseline"}  # also proves the detector sees imports
    assert oracle_imports(os.path.join(root, "__graft_entry__.py")) == set()  # smoke() reaches it through tests/step_parity.py only
