"""CPU test: libalva_b200.so loads without a GPU and exports every symbol include/alva_b200.h declares;
creating a context without a device fails loudly (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "alva_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(alva_[a-z0-9_]+)\s*\(", txt)))


def test_exports_every_declared_symbol():
    import alvaar_b200
    L = C.CDLL(alvaar_b200.lib_path())
    syms = declared_symbols()
    assert len(syms) >= 10
    missing = [s for s in syms if not hasattr(L, s)]
    assert not missing, f"declared in include/alva_b200.h but not exported: {missing}"


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import alvaar_b200
    with pytest.raises(alvaar_b200.AlvaError):
        alvaar_b200.Context(0)


def test_product_does_not_touch_oracle():
    """The product path may not import / link / execute anything under oracle/."""
    pkg = os.path.join(ROOT, "alvaar_b200")
    for dp, _, files in os.walk(pkg):
        if "_build" in dp:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")) or f == "Makefile":
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "libalva_oracle" not in txt and "libalva_ref" not in txt and "orc_" not in txt, (dp, f)


def test_reference_class_shim_compiles_and_links():
    """include/alva_system.hpp -- the reference's `class System` (system.hpp:28-38) over the C ABI, what embind.cpp binds --
    compiles with the reference's exact member signatures, links against the library and fails cleanly when unconfigured."""
    import subprocess
    import alvaar_b200
    out = os.path.join(ROOT, "tests", "_build", "system_shim_check")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    lib = alvaar_b200.lib_path()
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", out, os.path.join(ROOT, "tests", "host", "system_shim_check.cpp"), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    r = subprocess.run([out], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_python_system_binding_fails_loudly_without_a_gpu():
    """alvaar_b200.System (the ctypes mirror of the reference's class): without an sm_90 device configure() must raise -- never a
    silent CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import alvaar_b200
    with pytest.raises(alvaar_b200.AlvaError):
        alvaar_b200.System(640, 480, 500.0, 500.0, 320.0, 240.0)
