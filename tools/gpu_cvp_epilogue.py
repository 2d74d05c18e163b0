"""Times the CVP epilogue (k_cvp_epilogue, plus k_cvp_epilogue_csr where the build has it) by itself on the GPU and prints
one JSON line.

Workload: the bench plan -- the 5 M-vertex terrain (synth.grid_mesh(2240, 2240, terrain=True, seed=42)), the goal face of
bench.goal_for_rank(rank 0), a full-field mnb_cvp with all four outputs into device buffers.  Each library given with
--lib LABEL=PATH (default: the in-tree build as "tree") plans on its own MeshMap; the libraries take turns, --plans plans
each per turn, for --turns turns, under torch.profiler, which reads the kernels' device times.  Also reported per library:
the plan's CUDA-event kernel time (mnb_stats.kernel_ms) and whether its four output arrays are bit-identical to the first
library's.  The card's name, power limit and SM clock are read before and after.
Usage: python tools/gpu_cvp_epilogue.py [--lib LABEL=PATH ...] [--turns T] [--plans P] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except Exception as e:      # reported, not hidden
        return {"error": f"nvidia-smi: {e}"}


def load_lib(path):
    """the ctypes binding of the library at path (a library of its own next to any other loaded one)"""
    from mesh_navigation_b200 import _lib
    saved_path, saved = _lib.LIB_PATH, _lib._lib
    _lib.LIB_PATH, _lib._lib = path, None
    try:
        return _lib.load()
    finally:
        _lib.LIB_PATH, _lib._lib = saved_path, saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="LABEL=PATH of a libmeshnav_b200.so build (repeatable)")
    ap.add_argument("--size", type=int, default=2240)
    ap.add_argument("--turns", type=int, default=4)
    ap.add_argument("--plans", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("gpu_cvp_epilogue.py needs an H100")
    from bench import build_workload, goal_for_rank
    from mesh_navigation_b200 import _lib
    from mesh_navigation_b200.api import MeshMap

    libs = [tuple(x.split("=", 1)) for x in args.lib] or [("tree", _lib.LIB_PATH)]
    info_before = gpu_info()
    n = args.size
    pos, faces = build_workload(n)
    sf, sp = goal_for_rank(pos, faces, n, 0)
    runs = []
    for label, path in libs:
        _lib._lib = load_lib(os.path.abspath(path))       # MeshMap binds the library loaded last
        mm = MeshMap(pos, faces)
        ed = mm.edgeDistances(); mm.setCosts(np.zeros(mm.V, np.float32), ed)
        V = mm.V
        out = {"dist": torch.empty(V, dtype=torch.float32, device="cuda"), "pred": torch.empty(V, dtype=torch.int32, device="cuda"),
               "dir": torch.empty(V, dtype=torch.float32, device="cuda"), "cut": torch.empty(V, dtype=torch.int32, device="cuda")}
        runs.append({"label": label, "path": path, "mm": mm, "out": out, "epi_ms": [], "csr_ms": [], "grid_ms": [], "kernel_ms": []})
    _lib._lib = None

    def plan(r):
        mm = r["mm"]
        mm.use_device_pointers(True)
        o = r["out"]
        rc = mm.cvp_dev(sf, sp, -1, 1.0, 0.3, o["dist"].data_ptr(), o["pred"].data_ptr(), o["dir"].data_ptr(), o["cut"].data_ptr())
        mm.use_device_pointers(False)
        assert rc == 0, rc
        return mm.stats()

    for r in runs:                                          # warm-up
        for _ in range(2):
            plan(r)
    torch.cuda.synchronize()
    for _ in range(args.turns):
        for r in runs:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.plans):
                    r["kernel_ms"].append(plan(r)["kernel_ms"])
                torch.cuda.synchronize()
            epi, csr, grid = [], [], []
            for e in prof.events():
                if "k_cvp_epilogue_csr" in e.name:
                    csr.append(e.device_time_total / 1e3)
                elif "k_cvp_epilogue" in e.name:
                    epi.append(e.device_time_total / 1e3)
                elif "k_cvp_grid" in e.name:
                    grid.append(e.device_time_total / 1e3)
            assert len(epi) == args.plans, (r["label"], len(epi))
            r["epi_ms"] += epi; r["grid_ms"] += grid
            r["csr_ms"] += csr if csr else [0.0] * len(epi)
    ref = runs[0]["out"]
    res = []
    for r in runs:
        same = {k: bool(torch.equal(r["out"][k].view(torch.int32), ref[k].view(torch.int32))) for k in ref}
        e, c_ = np.array(r["epi_ms"]), np.array(r["csr_ms"])
        res.append({"label": r["label"], "epilogue_ms_median": float(np.median(e + c_)), "epilogue_ms_min": float((e + c_).min()),
                    "k_cvp_epilogue_ms_median": float(np.median(e)), "k_cvp_epilogue_csr_ms_median": float(np.median(c_)),
                    "k_cvp_grid_ms_median": float(np.median(r["grid_ms"])) if r["grid_ms"] else None,
                    "plan_kernel_ms_median": float(np.median(r["kernel_ms"])), "samples": int(e.size),
                    "identical_to_" + runs[0]["label"]: same})
        print(json.dumps(res[-1]), flush=True)
    for r in runs:
        r["mm"].close()
    line = {"tool": "gpu_cvp_epilogue", "V": int(runs[0]["mm"].V), "turns": args.turns,
            "plans_per_turn": args.plans, "gpu_before": info_before, "gpu_after": gpu_info(), "libs": res}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
