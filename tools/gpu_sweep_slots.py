"""Dev script (GPU box): GridStage slots per CTA x single-plan band width x in-round sweeps of the whole-grid kernels on the
bench plan (bench.py's 5 M terrain, goal of rank 0, cost limit 1, goal offset 0.3, L2 flushed before every plan).

For each (slots, band in mean edge weights w, sweeps) it prints the median kernel_ms of the timed plans (k_cvp_grid and the
epilogue, as bench.py times them), rounds, recomputes per vertex, and whether all four CVP outputs (Dijkstra: distances and
predecessors) are bit-identical to the first combination's.  The card, its power limit and SM clocks are printed first.

  python tools/gpu_sweep_slots.py cvp 1024:20:12,3072:40:24 [--size 2240] [--plans 5]
  python tools/gpu_sweep_slots.py dijkstra 1024:25:15,4096:40:24
slots 0 = the library default; band 0 = derived from the slots (mnb_set_costs); sweeps -1 = derived from the band."""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:    # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("kind", choices=["cvp", "dijkstra"])
    ap.add_argument("combos", help="slots:band_w:sweeps,...")
    ap.add_argument("--size", type=int, default=2240)
    ap.add_argument("--plans", type=int, default=5)
    args = ap.parse_args()
    import torch
    from bench import build_workload, goal_for_rank
    from mesh_navigation_b200.api import MeshMap

    print("card:", card(), flush=True)
    n = args.size
    pos, faces = build_workload(n)
    mm = MeshMap(pos, faces)
    ed = mm.edgeDistances()
    vc = np.zeros(mm.V, np.float32)
    fin = ed[(ed > 0) & np.isfinite(ed)].astype(np.float64)
    w = float(fin.sum() / fin.size)
    sf, sp = goal_for_rank(pos, faces, n, 0)
    seed = int(faces[sf][0])
    dev = torch.device("cuda", 0)
    outs = [torch.empty(mm.V, dtype=torch.int32, device=dev) for _ in range(4)]
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    for name in ("mnb_debug_set_sweeps", "mnb_debug_set_sweep_slots"):
        if hasattr(mm.L, name):               # (a build without the slots hook runs slots 0 only)
            getattr(mm.L, name).argtypes = [C.c_void_p, C.c_int32]
            getattr(mm.L, name).restype = C.c_int32

    def plan():
        flush.zero_()
        mm.use_device_pointers(True)
        if args.kind == "cvp":
            mm.cvp_dev(sf, sp, -1, 1.0, 0.3, *(o.data_ptr() for o in outs))
        else:
            mm.dijkstra_dev(seed, -1, 1e30, 0.0, outs[0].data_ptr(), outs[1].data_ptr())
        mm.use_device_pointers(False)
        return mm.stats()

    ref = None
    print(f"V={mm.V} w={w:.5f} hop=1.35w", flush=True)
    for c in args.combos.split(","):
        slots, band, sweeps = c.split(":")
        slots, band, sweeps = int(slots), float(band), int(sweeps)
        if slots or hasattr(mm.L, "mnb_debug_set_sweep_slots"):
            assert mm.L.mnb_debug_set_sweep_slots(mm._ctx, slots) == 0, f"slots {slots} do not fit"
        mm.setCosts(vc, ed)                           # band widths derived from the slots (unless explicit below)
        if band > 0:
            mm.set_tuning(band * w, 0, 0)
        assert mm.L.mnb_debug_set_sweeps(mm._ctx, sweeps) == 0
        plan()
        ms = []
        for _ in range(args.plans):
            st = plan()
            ms.append(st["kernel_ms"])
        torch.cuda.synchronize()
        got = [o.cpu().numpy().copy() for o in outs[: 4 if args.kind == "cvp" else 2]]
        if ref is None:
            ref = got
        same = all((g == r).all() for g, r in zip(got, ref))
        print(f"{args.kind} slots={slots} band={band:g}w sweeps={sweeps}: kernel_ms median {np.median(ms):.3f} "
              f"(min {min(ms):.3f} max {max(ms):.3f}) rounds={st['rounds']} recomp/V={st['recomputes'] / mm.V:.3f} "
              f"bit-equal={same}", flush=True)
    mm.close()


if __name__ == "__main__":
    main()
