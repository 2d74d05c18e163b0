"""Runs pytest on the GPU parity suite with the ctypes binding pointed at tests/emu/libmeshnav_emu.so.

Test infrastructure: the CUDA kernels' sources, compiled unchanged by g++ against the CPU interpreter in this directory,
are driven through the same C ABI and compared with the oracle exactly as `-m gpu` does on an H100 (small meshes only).
Usage: python tests/emu/run_suite.py <pytest args>"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def build():
    subprocess.check_call(["make", "-s", "-C", HERE])
    return os.path.join(HERE, "libmeshnav_emu.so")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    os.chdir(ROOT)
    lib = build()
    from mesh_navigation_b200 import _lib
    _lib.LIB_PATH = lib          # the interpreter exports the same C ABI; only this test driver ever points here
    import pytest
    sys.exit(pytest.main(sys.argv[1:]))
