"""Dry-run of bench.py's GPU arm on the CPU interpreter of the kernels (tiny sizes, one emulated SM so that every launch
runs in this process and may write to ordinary host memory).  torch's CUDA entry points are stubbed: "device" tensors are
host tensors.  Purpose: execute every line of the bench orchestration (legs, JSON assembly) before it meets a real GPU;
the numbers it prints mean nothing.   usage: python tests/emu/run_bench_on_emu.py [bench args]"""
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
os.environ["MNB_EMU_SMS"] = "1"
from tests.emu.run_suite import build  # noqa: E402

from mesh_navigation_b200 import _lib  # noqa: E402
_lib.LIB_PATH = build()
import torch  # noqa: E402

torch.cuda.is_available = lambda: True
torch.cuda.set_device = lambda *a, **k: None
torch.cuda.synchronize = lambda *a, **k: None
_empty, _tensor, _device = torch.empty, torch.tensor, torch.device
torch.device = lambda *a, **k: _device("cpu")
torch.empty = lambda *a, **k: _empty(*a, **{kk: vv for kk, vv in k.items() if kk != "device"})
torch.tensor = lambda *a, **k: _tensor(*a, **{kk: vv for kk, vv in k.items() if kk != "device"})
torch.Tensor.pin_memory = lambda self, *a, **k: self

if __name__ == "__main__":
    args = sys.argv[1:] or ["--size", "120", "--batch-size", "60", "--batch-goals", "6", "--batch-steps", "1", "--steps", "2", "--warmup", "1"]
    sys.argv = [os.path.join(ROOT, "bench.py")] + args
    runpy.run_path(os.path.join(ROOT, "bench.py"), run_name="__main__")
