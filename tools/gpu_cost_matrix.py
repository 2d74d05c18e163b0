"""Measures the cost-matrix calls (mnb_dijkstra_matrix / mnb_cvp_matrix) on the GPU and prints one JSON line.

Every leg checks the matrix bit for bit against the gathered rows of the batch call with the same seeds.
Spread: the 1 M-vertex terrain (synth.grid_mesh(1000, 1000, terrain=True)), the config-4 goals
(synth.batch_goal_vertices(V, 1024, seed=1234)) and 256 targets spread over the map (seed 77).  Timed alternately call by
call in one process: the matrix into a device [n, m] buffer, and the batch into device [n, V] rows plus a torch gather.
Reported for Dijkstra and CVP: plans/s, kernel time, and the device memory each call grows on a fresh map in host-pointer
mode (workspace plus the library's device staging of the output).
Local: seeds and targets drawn from one 100 x 100-vertex window (10 m x 10 m) of the same terrain.  Reported: plans/s,
settled vertices per wave (matrix and batch), kernel time, and the workspace bytes every call clears (V x bytes per
vertex x goals: computed, not timed).
Large: the 5 M-vertex terrain, 256 goals, CVP: the concurrent waves the free-memory cap allows the matrix and
mnb_cvp_batch with host rows, from the growth of the device memory over a fresh map.
Usage: python tools/gpu_cost_matrix.py [--steps K] [--warmup W]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WS_CLEARED_BYTES_PER_VERTEX = {"dijkstra": 16, "cvp": 40}     # written per vertex before each goal (label, mark, lists / state, mark, chg, skip words)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except Exception as e:      # reported, not hidden
        return {"error": f"nvidia-smi: {e}"}


def used_bytes(torch):
    free, total = torch.cuda.mem_get_info()
    return total - free


def ws_per_wave(kind, V):
    """ensure_workspace / the Dijkstra batch workspace, without the GroupCtl"""
    return 16 * V if kind == "dijkstra" else 56 * V + 4 * max(65536, 2 * V)


def make_map(n):
    from mesh_navigation_b200 import synth
    from mesh_navigation_b200.api import MeshMap
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=42)
    mm = MeshMap(pos, faces)
    mm.setCosts(np.zeros(mm.V, np.float32), mm.edgeDistances())
    return pos, faces, mm


def goal_faces(pos, faces, n, vertices):
    gi, gj = np.minimum(vertices % n, n - 2), np.minimum(vertices // n, n - 2)
    sfs = (2 * (gj * (n - 1) + gi)).astype(np.uint32)
    return sfs, pos[faces[sfs]].mean(1).astype(np.float32)


class Calls:
    """the matrix and the batch + gather of one planner kind, device pointers; every call ends in a stream synchronise"""

    def __init__(self, torch, mm, kind, seeds, sfs, sps, targets):
        self.torch, self.mm, self.kind, self.seeds, self.sfs, self.sps = torch, mm, kind, seeds, sfs, sps
        self.targets = targets
        self.t_idx = torch.from_numpy(targets.astype(np.int64)).cuda()
        self.n = seeds.size

    def matrix(self, out):
        if self.kind == "dijkstra":
            assert self.mm.dijkstra_matrix_dev(self.seeds, self.targets, 1.0, out.data_ptr()) == 0
        else:
            assert self.mm.cvp_matrix_dev(self.sfs, self.sps, self.targets, 1.0, out.data_ptr()) == 0
        return self.mm.stats()

    def batch(self, rows):
        if self.kind == "dijkstra":
            assert self.mm.dijkstra_batch_dev(self.seeds, 1.0, rows.data_ptr()) == 0
        else:
            assert self.mm.cvp_batch_dev(self.sfs, self.sps, 1.0, rows.data_ptr()) == 0
        st = self.mm.stats()
        g = rows.index_select(1, self.t_idx)
        self.torch.cuda.synchronize()
        return st, g


def fresh_growth(torch, n, kind, seeds, sfs, sps, targets):
    """device memory grown by one matrix call and one batch call, each on a fresh map in host-pointer mode"""
    from mesh_navigation_b200.api import CVPMeshPlanner, DijkstraMeshPlanner
    res = {}
    for what in ("matrix", "batch"):
        _, _, mm = make_map(n)
        pl = DijkstraMeshPlanner(mm) if kind == "dijkstra" else CVPMeshPlanner(mm)
        args = (seeds,) if kind == "dijkstra" else (sfs, sps)
        u0 = used_bytes(torch)
        if what == "matrix":
            r = pl.costMatrix(*args, targets)
        else:
            r = pl.dijkstraBatch(seeds, want_pred=False) if kind == "dijkstra" else pl.waveFrontPropagationBatch(sfs, sps)
        res[what] = int(used_bytes(torch) - u0)
        assert r["outcome"] == 0
        del r
        mm.close()
        torch.cuda.empty_cache()
    res["workspace_bytes_per_wave"] = ws_per_wave(kind, n * n)
    res["batch_staging_rows_bytes"] = 4 * seeds.size * n * n
    res["matrix_staging_bytes"] = 4 * seeds.size * targets.size
    return res


def timed_pair(torch, calls, steps, warmup):
    """matrix vs batch + gather, alternated call by call"""
    V = calls.mm.V
    out = torch.empty((calls.n, calls.targets.size), dtype=torch.float32, device="cuda")
    rows = torch.empty((calls.n, V), dtype=torch.float32, device="cuda")
    st_m = calls.matrix(out)
    st_b, g = calls.batch(rows)
    exact = bool((out.view(torch.int32) == g.view(torch.int32)).all().item())
    for _ in range(warmup):
        calls.matrix(out); calls.batch(rows)
    tm, tb, km, kb = [], [], [], []
    for _ in range(steps):
        t0 = time.perf_counter(); st_m = calls.matrix(out); tm.append(time.perf_counter() - t0); km.append(st_m["kernel_ms"])
        t0 = time.perf_counter(); st_b, g = calls.batch(rows); tb.append(time.perf_counter() - t0); kb.append(st_b["kernel_ms"])
    exact = exact and bool((out.view(torch.int32) == g.view(torch.int32)).all().item())
    n = calls.n
    res = {"goals": int(n), "targets": int(calls.targets.size), "entries_bit_identical_to_gathered_rows": exact,
           "matrix": {"plans_per_s": n / float(np.mean(tm)), "s_per_call": float(np.mean(tm)), "kernel_s_mean": float(np.mean(km)) / 1e3,
                      "kernel_s_min": float(np.min(km)) / 1e3, "settled_per_wave": st_m["settled"] / n, "rounds_per_wave": st_m["rounds"] / n},
           "batch_plus_gather": {"plans_per_s": n / float(np.mean(tb)), "s_per_call": float(np.mean(tb)), "kernel_s_mean": float(np.mean(kb)) / 1e3,
                                 "kernel_s_min": float(np.min(kb)) / 1e3, "settled_per_wave": st_b["settled"] / n, "rounds_per_wave": st_b["rounds"] / n},
           "workspace_bytes_cleared_per_call": int(V * WS_CLEARED_BYTES_PER_VERTEX[calls.kind] * n),
           "steps": steps, "warmup": warmup}
    del rows
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3, help="timed calls of each kind (alternated)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--size", type=int, default=1000)
    ap.add_argument("--goals", type=int, default=1024)
    ap.add_argument("--targets", type=int, default=256)
    ap.add_argument("--window", type=int, default=100, help="local leg: side of the vertex window seeds and targets come from")
    ap.add_argument("--large-size", type=int, default=2236, help="large leg grid side (2236 -> 5 M vertices); 0 skips it")
    ap.add_argument("--large-goals", type=int, default=256)
    args = ap.parse_args()
    import torch
    from mesh_navigation_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU mode")
    res = {"tool": "gpu_cost_matrix", "gpu": gpu_info()}
    n = args.size

    # ---- spread and local legs: 1 M terrain --------------------------------------------------------------------------
    pos, faces, mm = make_map(n)
    V = mm.V
    mm.use_device_pointers(True)
    seeds = synth.batch_goal_vertices(V, args.goals, seed=1234).astype(np.uint32)
    targets = synth.batch_goal_vertices(V, args.targets, seed=77).astype(np.uint32)
    sfs, sps = goal_faces(pos, faces, n, seeds)
    rng = np.random.default_rng(5)
    w0 = (n - args.window) // 2
    i, j = np.meshgrid(np.arange(w0, w0 + args.window), np.arange(w0, w0 + args.window))
    window = (j * n + i).ravel()
    lseeds = rng.choice(window, args.goals, replace=False).astype(np.uint32)
    ltargets = rng.choice(window, args.targets, replace=False).astype(np.uint32)
    lsfs, lsps = goal_faces(pos, faces, n, lseeds)
    for kind in ("dijkstra", "cvp"):
        res[f"spread_{kind}_1m"] = timed_pair(torch, Calls(torch, mm, kind, seeds, sfs, sps, targets), args.steps, args.warmup)
        res[f"local_{kind}_1m"] = timed_pair(torch, Calls(torch, mm, kind, lseeds, lsfs, lsps, ltargets), args.steps, args.warmup)
        res[f"local_{kind}_1m"]["window"] = f"{args.window} x {args.window} vertices at ({w0}, {w0})"
    res["mesh_vertices_1m"] = int(V)
    res["gpu_after_timing"] = gpu_info()
    mm.close()
    torch.cuda.empty_cache()
    for kind in ("dijkstra", "cvp"):
        res[f"spread_{kind}_1m"]["device_memory_grown_bytes_host_mode"] = fresh_growth(torch, n, kind, seeds, sfs, sps, targets)

    # ---- large leg: 5 M terrain, CVP, concurrent waves under the memory cap -------------------------------------------
    if args.large_size > 0:
        nl = args.large_size
        leg = {"goals": args.large_goals}
        from mesh_navigation_b200.api import CVPMeshPlanner
        cost = None
        for what in ("matrix", "batch_host_rows"):
            pos, faces, mm = make_map(nl)            # a fresh map: its workspace grows from nothing
            V = mm.V
            g = synth.batch_goal_vertices(V, args.large_goals, seed=1234).astype(np.uint32)
            sfs, sps = goal_faces(pos, faces, nl, g)
            tg = synth.batch_goal_vertices(V, args.targets, seed=77).astype(np.uint32)
            pl = CVPMeshPlanner(mm)
            u0 = used_bytes(torch)
            t0 = time.perf_counter()
            if what == "matrix":
                r = pl.costMatrix(sfs, sps, tg)
                cost = r["cost"]
                staging = 4 * sfs.size * tg.size
            else:
                r = pl.waveFrontPropagationBatch(sfs, sps)
                leg["entries_bit_identical_to_gathered_rows"] = bool((r["dist"][:, tg].view(np.uint32) == cost.view(np.uint32)).all())
                staging = 4 * sfs.size * V
                del r["dist"]
            t1 = time.perf_counter() - t0
            grown = used_bytes(torch) - u0
            leg[what] = {"device_memory_grown_bytes": int(grown), "staging_bytes": int(staging),
                         "concurrent_waves_from_workspace": int((grown - staging) // (ws_per_wave("cvp", V) + 256)),
                         "s_per_call": t1, "kernel_s": r["kernel_ms"] / 1e3, "settled_per_wave": r["settled"] / sfs.size}
            leg["mesh_vertices"] = int(V)
            mm.close()
            torch.cuda.empty_cache()
        res["large_cvp_5m"] = leg
    res["gpu_end"] = gpu_info()
    res["all_entries_exact"] = all(v.get("entries_bit_identical_to_gathered_rows", True) for v in res.values() if isinstance(v, dict))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
