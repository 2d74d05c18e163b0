"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol the header
declares, and FAILS LOUDLY (no fallback) when no sm_90 device is present."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    txt = open(os.path.join(ROOT, "include", "meshnav_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(mnb_[a-z_0-9]+)\s*\(", txt)))


def test_header_symbols_exported():
    from mesh_navigation_b200 import _lib
    L = _lib.load()
    names = header_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/meshnav_b200.h but not exported"
    assert sorted(_lib.EXPORTS) == names


def test_no_cpu_fallback_without_gpu():
    """Without a usable sm_90 device mnb_create must fail (MNB_E_CUDA) -- nothing routes to a CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the loud-failure path is exercised on the CPU-only build box")
    from mesh_navigation_b200 import _lib
    from mesh_navigation_b200.api import MeshMap, MeshNavError
    L = _lib.load()
    ctx = C.c_void_p()
    assert L.mnb_create(0, C.byref(ctx)) == -2 and not ctx.value
    pos = np.zeros((3, 3), np.float32); faces = np.array([[0, 1, 2]], np.uint32)
    with pytest.raises(MeshNavError):
        MeshMap(pos, faces)


def test_product_never_imports_oracle():
    """The product package and the CUDA sources must not reference oracle/ (parity claims depend on it)."""
    pkg = os.path.join(ROOT, "mesh_navigation_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src and "liboracle" not in src, f


def test_product_never_loads_the_cpu_interpreter():
    """tests/emu (the CPU interpreter of the kernels, test infrastructure) must stay out of the product: the package never
    names it, and the shipped library contains no interpreter symbols (MNB_EMU_ACTIVE is only defined by tests/emu)."""
    pkg = os.path.join(ROOT, "mesh_navigation_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "libmeshnav_emu" not in src and "tests.emu" not in src and "tests/emu" not in src, f
    blob = open(os.path.join(pkg, "libmeshnav_b200.so"), "rb").read()
    assert b"mnb_emu_switch" not in blob and b"mnb-emu" not in blob
    assert b"sm_90a" in blob, "the shipped library carries no sm_90a code"
