"""Measures the batched full-field Dijkstra planner (mnb_dijkstra_batch) on the GPU and prints one JSON line.

Leg 1: the 1 M-vertex terrain (synth.grid_mesh(1000, 1000, terrain=True)), the config-4 goal set
(synth.batch_goal_vertices(V, 1024, seed=1234)), distances + predecessors into device buffers.  Reported: plans/s, kernel
time, settled vertices/s and the algorithmic bandwidth (92 B per settled vertex) against the 3.35 TB/s data sheet; the same
goals as a loop of single mnb_dijkstra calls (timed on a sample, extrapolated); the single-core oracle per plan; 8 rows
checked bit for bit against the oracle.
Leg 2: the 5 M-vertex terrain, 256 goals, distances only, with part of the device memory held by a ballast tensor so that
the free-memory cap of the concurrent wavefronts binds.
Usage: python tools/gpu_dijkstra_batch.py [--steps K] [--warmup W] [--sweep-delta-w 1,2.5,5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BYTES_PER_SETTLED = 92          # DESIGN §5: one Dijkstra relaxation sweep over a settled vertex's CSR row + label traffic
HBM_PEAK_GBS = 3350.0           # H100 SXM data sheet (HBM3), not a measured figure
WS_BYTES_PER_VERTEX = 16        # k_dijkstra_batch: float label + mark + two candidate lists


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


def setup(n):
    from mesh_navigation_b200 import synth
    from mesh_navigation_b200.api import MeshMap
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=42)
    mm = MeshMap(pos, faces)
    ed = mm.edgeDistances(); vc = np.zeros(mm.V, np.float32)
    mm.setCosts(vc, ed)
    return pos, faces, mm, ed, vc


def timed_batch(mm, goals, d_dist, d_pred, steps, warmup):
    for _ in range(warmup):
        mm.dijkstra_batch_dev(goals, 1.0, d_dist, d_pred)
    kms, st = [], None
    t0 = time.perf_counter()
    for _ in range(steps):
        assert mm.dijkstra_batch_dev(goals, 1.0, d_dist, d_pred) == 0
        st = mm.stats(); kms.append(st["kernel_ms"])      # every call ends in a stream synchronise
    wall = time.perf_counter() - t0
    return wall / steps, float(np.mean(kms)), float(np.min(kms)), st


def parity(om, w, vc, goals, rows, d_dist, d_pred):
    bad = []
    for k in rows:
        ref = om.dijkstra(w, vc, int(goals[k]))
        dist = d_dist[k].cpu().numpy()
        ok = (dist.view(np.uint32) == ref["dist"].view(np.uint32)).all()
        if d_pred is not None:
            ok = ok and (d_pred[k].cpu().numpy().view(np.uint32) == ref["pred"]).all()
        if not ok:
            bad.append(int(k))
    return {"rows_checked": [int(k) for k in rows], "mismatching_rows": bad, "ok": not bad}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--goals", type=int, default=1024)
    ap.add_argument("--size", type=int, default=1000)
    ap.add_argument("--single-sample", type=int, default=64)
    ap.add_argument("--large-size", type=int, default=2236, help="leg 2 grid side (2236 -> 5 M vertices); 0 skips leg 2")
    ap.add_argument("--large-goals", type=int, default=256)
    ap.add_argument("--large-free-gb", type=float, default=12.0, help="leg 2: device memory left free next to the ballast")
    ap.add_argument("--sweep-delta-w", default="", help="comma-separated band widths in mean edge weights to time after leg 1")
    args = ap.parse_args()
    import torch
    from oracle import oracle as O
    from mesh_navigation_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU mode")
    res = {"tool": "gpu_dijkstra_batch", "gpu": gpu_info()}

    # ---- leg 1: 1 M terrain, 1024 goals, dist + pred --------------------------------------------------------------
    pos, faces, mm, ed, vc = setup(args.size)
    V = mm.V
    goals = synth.batch_goal_vertices(V, args.goals, seed=1234).astype(np.uint32)
    d_dist = torch.empty((goals.size, V), dtype=torch.float32, device="cuda")
    d_pred = torch.empty((goals.size, V), dtype=torch.int32, device="cuda")
    mm.use_device_pointers(True)
    used0 = used_bytes(torch)
    mm.dijkstra_batch_dev(goals, 1.0, d_dist.data_ptr(), d_pred.data_ptr())
    ws_bytes = used_bytes(torch) - used0          # the workspace stays allocated after the call
    per_call, kms_mean, kms_min, st = timed_batch(mm, goals, d_dist.data_ptr(), d_pred.data_ptr(), args.steps, args.warmup)
    gpu_during = gpu_info()
    settled = st["settled"]
    batch = {"mesh_vertices": int(V), "goals": int(goals.size), "outputs": "dist + pred, device pointers",
             "plans_per_s": goals.size / per_call, "ms_per_call": 1e3 * per_call, "kernel_ms_mean": kms_mean, "kernel_ms_min": kms_min,
             "rounds_summed_over_wavefronts": int(st["rounds"]), "settled": int(settled),
             "settled_vertices_per_s": settled / (kms_mean * 1e-3),
             "achieved_gbs_at_92B_per_settled_vertex": BYTES_PER_SETTLED * settled / (kms_mean * 1e-3) / 1e9,
             "hbm_datasheet_gbs": HBM_PEAK_GBS,
             "workspace_bytes_from_device_memory_growth": int(ws_bytes),
             "wavefronts_in_flight_from_workspace": int(ws_bytes // (WS_BYTES_PER_VERTEX * V)),
             "device_memory_in_use_bytes": int(used_bytes(torch)), "steps": args.steps, "warmup": args.warmup}
    batch["hbm_frac_of_datasheet"] = batch["achieved_gbs_at_92B_per_settled_vertex"] / HBM_PEAK_GBS
    res["batch_1m"] = batch
    # the same goals as single mnb_dijkstra calls (whole-grid kernel), timed on a sample and extrapolated
    sd = torch.empty(V, dtype=torch.float32, device="cuda"); sp = torch.empty(V, dtype=torch.int32, device="cuda")
    sample = goals[: args.single_sample]
    for s in sample[:2]:
        mm.dijkstra_dev(int(s), -1, 1.0, 0.3, sd.data_ptr(), sp.data_ptr())
    single_k = []
    t0 = time.perf_counter()
    for s in sample:
        mm.dijkstra_dev(int(s), -1, 1.0, 0.3, sd.data_ptr(), sp.data_ptr())
        single_k.append(mm.stats()["kernel_ms"])
    t_single = (time.perf_counter() - t0) / sample.size
    res["single_loop_1m"] = {"sampled_goals": int(sample.size), "ms_per_plan": 1e3 * t_single, "kernel_ms_per_plan": float(np.mean(single_k)),
                             "plans_per_s": 1.0 / t_single, "extrapolated_ms_for_all_goals": 1e3 * t_single * goals.size,
                             "note": "loop of mnb_dijkstra(seed, -1) on a sample of the goals, extrapolated to the whole set"}
    res["batch_vs_single_loop"] = batch["plans_per_s"] / res["single_loop_1m"]["plans_per_s"]
    # parity: 8 sampled rows against the oracle (the first 4 also time the oracle per plan)
    om =O.OracleMesh(pos, faces)
    rows = np.unique(np.linspace(0, goals.size - 1, 8).astype(np.int64))
    t_or = []
    for k in rows[:4]:
        t_or.append(om.dijkstra(ed, vc, int(goals[k]))["seconds"])
    res["oracle_1core_s_per_plan"] = float(np.mean(t_or))
    res["parity_1m"] = parity(om, ed, vc, goals, rows, d_dist, d_pred)
    if args.sweep_delta_w:
        wm = float(ed[np.isfinite(ed)].astype(np.float64).mean())
        sweep = {}
        for k in [float(x) for x in args.sweep_delta_w.split(",")]:
            mm.set_tuning(k * wm, 0, 0)
            pc, km, _, s2 = timed_batch(mm, goals, d_dist.data_ptr(), d_pred.data_ptr(), max(1, args.steps // 2), 1)
            sweep[str(k)] = {"plans_per_s": goals.size / pc, "kernel_ms": km, "rounds_summed": int(s2["rounds"]),
                             "recomputes_per_settled": s2["recomputes"] / max(1, s2["settled"])}
        res["band_sweep_1m_delta_in_mean_edge_weights"] = sweep
        res["parity_1m_after_sweep"] = parity(om, ed, vc, goals, rows[:2], d_dist, d_pred)
    mm.use_device_pointers(False)
    mm.close(); del d_dist, d_pred, sd, sp, om
    torch.cuda.empty_cache()

    # ---- leg 2: 5 M terrain, 256 goals, dist only, with the memory cap binding ------------------------------------
    if args.large_size > 0:
        pos, faces, mm, ed, vc = setup(args.large_size)
        V = mm.V
        goals = synth.batch_goal_vertices(V, args.large_goals, seed=1234).astype(np.uint32)
        d_dist = torch.empty((goals.size, V), dtype=torch.float32, device="cuda")
        free, total = torch.cuda.mem_get_info()
        ballast_bytes = max(0, int(free - args.large_free_gb * 2**30))
        ballast = torch.empty(ballast_bytes, dtype=torch.uint8, device="cuda")
        mm.use_device_pointers(True)
        used0 = used_bytes(torch)
        t0 = time.perf_counter()
        rc = mm.dijkstra_batch_dev(goals, 1.0, d_dist.data_ptr(), 0)
        t1 = time.perf_counter() - t0
        ws = used_bytes(torch) - used0
        st = mm.stats()
        leg = {"mesh_vertices": int(V), "goals": int(goals.size), "outputs": "dist only, device pointers", "outcome": rc,
               "ballast_bytes": ballast_bytes, "free_bytes_before_call": int(total - used0),
               "workspace_bytes_from_device_memory_growth": int(ws), "wavefronts_in_flight_from_workspace": int(ws // (WS_BYTES_PER_VERTEX * V)),
               "wavefronts_without_the_cap": "min(goals, CTA slots) = min(%d, SMs x 4)" % goals.size,
               "ms_per_call": 1e3 * t1, "kernel_ms": st["kernel_ms"], "plans_per_s": goals.size / t1,
               "device_memory_in_use_bytes": int(used_bytes(torch))}
        mm.use_device_pointers(False)
        del ballast
        om = O.OracleMesh(pos, faces)
        leg["parity"] = parity(om, ed, vc, goals, [0, goals.size - 1], d_dist, None)
        res["batch_5m_memory_capped"] = leg
        mm.close()
    res["gpu_after_timing"] = gpu_during
    ok = res["parity_1m"]["ok"] and res.get("batch_5m_memory_capped", {}).get("parity", {"ok": True})["ok"]
    res["parity_ok"] = bool(ok and res.get("parity_1m_after_sweep", {"ok": True})["ok"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
