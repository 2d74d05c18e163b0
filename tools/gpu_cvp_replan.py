"""Measures CVP replanning (mnb_cvp_replan) against a fresh mnb_cvp on the GPU and prints one JSON line.

The map is the bench's 5 M-vertex terrain (2240 x 2240, 0.1 m) with zero costs and the edge weights of edge_cost_factor 1;
the goal (the wave's seed) is the face at the centre.  For each robot distance (along the diagonal) the change is a ring of
raised costs (0.5, cost limit 1) between 2 and 5 m around the robot, applied and removed again through
mnb_update_vertex_costs, so consecutive calls alternate between two cost sets.  Each workload runs the full field (robot
face -1) and with the robot cutoff.  Per call, the fresh plan and the replan run on the same costs in the same process,
alternated, with device outputs (torch tensors); every replan's four rows are checked bit for bit against the fresh plan.
Times: the CUDA-event time the library reports (kernel_ms) and the host clock around the call; medians over the timed
calls after one untimed round.  A separate torch.profiler run of one replan per workload gives the kernel times of the
O(V) passes (T0 reduction, rollback, frontier, epilogue).
Usage: python tools/gpu_cvp_replan.py [--reps N] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except Exception as e:      # reported, not hidden
        return {"error": f"nvidia-smi: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--n", type=int, default=2240)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from mesh_navigation_b200 import synth
    from mesh_navigation_b200.api import CVPMeshPlanner, MeshMap
    n = args.n
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=42)
    mm = MeshMap(pos, faces)
    V = mm.V
    vc = np.zeros(V, np.float32)
    mm.computeEdgeWeights(vc, 1.0, want_output=False)
    pl = CVPMeshPlanner(mm, cost_limit=1.0, goal_dist_offset=0.3)
    c = n // 2
    sf = 2 * (c * (n - 1) + c)
    sp = pos[faces[sf]].mean(0).astype(np.float32)
    dev = [torch.empty(V, dtype=t, device="cuda") for t in (torch.float32, torch.int32, torch.float32, torch.int32)]
    ref = [torch.empty(V, dtype=t, device="cuda") for t in (torch.float32, torch.int32, torch.float32, torch.int32)]
    mm.use_device_pointers(True)
    results = []
    h = 0.1
    for dist_m in (10.0, 30.0, 60.0, 100.0):
        k = int(round(dist_m / np.sqrt(2) / h))
        ri = min(n - 2, c + k)
        rf = 2 * (ri * (n - 1) + ri)
        rxy = pos[faces[rf]].mean(0)[:2]
        d = np.linalg.norm(pos[:, :2] - rxy[None, :], axis=1)
        ring = np.where((d >= 2.0) & (d <= 5.0))[0].astype(np.uint32)
        ring_d = torch.from_numpy(ring.view(np.int32)).cuda()
        hi = torch.full((ring.size,), 0.5, dtype=torch.float32, device="cuda")
        lo = torch.zeros(ring.size, dtype=torch.float32, device="cuda")
        for robot in (-1, rf):
            fresh_ms, replan_ms, fresh_wall, replan_wall, stats = [], [], [], [], []
            vals = [hi, lo]
            # the resident wave of this workload's seed and robot
            assert mm.cvp_replan_dev(sf, sp, robot, 1.0, 0.3, ring[:0], *[x.data_ptr() for x in dev]) in (0, 54)
            for it in range(args.reps + 1):
                mm.layerChanged((ring_d.data_ptr(), ring.size), vals[it % 2].data_ptr(), 1.0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rc_f = mm.cvp_dev(sf, sp, robot, 1.0, 0.3, *[x.data_ptr() for x in ref])
                t1 = time.perf_counter()
                sf_stats = mm.stats()
                t2 = time.perf_counter()
                rc_r = mm.cvp_replan_dev(sf, sp, robot, 1.0, 0.3, ring, *[x.data_ptr() for x in dev])
                t3 = time.perf_counter()
                sr_stats = mm.stats()
                assert rc_f == rc_r, (rc_f, rc_r)
                for a, b in zip(dev, ref):
                    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "replan differs from mnb_cvp"
                if it == 0:
                    continue
                fresh_ms.append(sf_stats["kernel_ms"]); replan_ms.append(sr_stats["kernel_ms"])
                fresh_wall.append(1e3 * (t1 - t0)); replan_wall.append(1e3 * (t3 - t2))
                stats.append((sf_stats["rounds"], sr_stats["rounds"], sf_stats["settled"], sr_stats["settled"]))
            # kernel times of the passes of one replan (profiler in a run of its own)
            mm.layerChanged((ring_d.data_ptr(), ring.size), vals[(args.reps + 1) % 2].data_ptr(), 1.0)
            torch.cuda.synchronize()
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                mm.cvp_replan_dev(sf, sp, robot, 1.0, 0.3, ring, *[x.data_ptr() for x in dev])
                torch.cuda.synchronize()
            kt = {}
            for e in prof.events():
                for key in ("k_replan_t0_final", "k_replan_t0", "k_replan_rollback", "k_replan_frontier", "k_cvp_epilogue", "k_cvp_grid"):
                    if key in e.name:
                        kt[key] = kt.get(key, 0.0) + e.device_time_total / 1e3
                        break
            st = np.array(stats, dtype=np.float64)
            results.append({
                "robot_dist_m": dist_m, "robot_face": int(robot), "ring_vertices": int(ring.size),
                "fresh_kernel_ms": float(np.median(fresh_ms)), "replan_kernel_ms": float(np.median(replan_ms)),
                "fresh_wall_ms": float(np.median(fresh_wall)), "replan_wall_ms": float(np.median(replan_wall)),
                "rounds_fresh": float(np.median(st[:, 0])), "rounds_replan": float(np.median(st[:, 1])),
                "settled_fresh": float(np.median(st[:, 2])), "settled_replan": float(np.median(st[:, 3])),
                "settled_share": float(np.median(st[:, 3] / np.maximum(st[:, 2], 1))),
                "replan_pass_ms": kt,
            })
            print(json.dumps(results[-1]), flush=True)
    mm.use_device_pointers(False)
    line = {"tool": "gpu_cvp_replan", "V": int(V), "reps": args.reps, "gpu": gpu_info(), "workloads": results, "exact": True}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
