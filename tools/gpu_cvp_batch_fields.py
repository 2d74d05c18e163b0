"""Measures the batched CVP vector fields (mnb_cvp_batch_fields) on the GPU and prints one JSON line.

Leg 1: the 1 M-vertex terrain (synth.grid_mesh(1000, 1000, terrain=True)), the config-4 goal set
(synth.batch_goal_vertices(V, 1024, seed=1234), the grid face at each goal vertex, its centroid as the goal point), into
device buffers.  Timed alternately in the same process: all four outputs through mnb_cvp_batch_fields, and the potentials
alone through mnb_cvp_batch -- their difference is the cost of the per-wave epilogue.  Also: a loop of single full-field
mnb_cvp calls on a sample of the goals (extrapolated), workspace and output bytes, the wavefront count, and 8 sampled
rows checked against the oracle and against single mnb_cvp.
Leg 2: the 5 M-vertex terrain, 64 goals, all four outputs, with part of the device memory held by a ballast tensor so that
the free-memory cap of the concurrent wavefronts binds; 2 rows checked against the oracle.
Usage: python tools/gpu_cvp_batch_fields.py [--steps K] [--warmup W]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KEYS = ("dist", "pred", "direction", "cutting_face")


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


def setup(n, n_goals):
    from mesh_navigation_b200 import synth
    from mesh_navigation_b200.api import MeshMap
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=42)
    mm = MeshMap(pos, faces)
    ed = mm.edgeDistances(); vc = np.zeros(mm.V, np.float32)
    mm.setCosts(vc, ed)
    goals = synth.batch_goal_vertices(mm.V, n_goals, seed=1234)
    gi, gj = np.minimum(goals % n, n - 2), np.minimum(goals // n, n - 2)
    sfs = (2 * (gj * (n - 1) + gi)).astype(np.uint32)
    sps = pos[faces[sfs]].mean(1).astype(np.float32)
    return pos, faces, mm, ed, vc, sfs, sps


def outputs(torch, n, V):
    return {"dist": torch.empty((n, V), dtype=torch.float32, device="cuda"), "pred": torch.empty((n, V), dtype=torch.int32, device="cuda"),
            "direction": torch.empty((n, V), dtype=torch.float32, device="cuda"),
            "cutting_face": torch.empty((n, V), dtype=torch.int32, device="cuda")}


def fields_call(mm, sfs, sps, bufs):
    assert mm.cvp_batch_fields_dev(sfs, sps, 1.0, *[bufs[k].data_ptr() for k in KEYS]) == 0
    return mm.stats()               # every call ends in a stream synchronise


def dist_call(mm, sfs, sps, bufs):
    assert mm.cvp_batch_dev(sfs, sps, 1.0, bufs["dist"].data_ptr()) == 0
    return mm.stats()


def parity(om, ed, vc, sfs, sps, rows, bufs, single=None):
    bad = []
    for k in rows:
        ref = om.cvp(ed, vc, int(sfs[k]), sps[k])
        got = {key: bufs[key][k].cpu().numpy() for key in KEYS}
        ok = (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
        ok = ok and (got["pred"].view(np.uint32) == ref["pred"]).all() and (got["cutting_face"] == ref["cutting_face"]).all()
        ok = ok and float(np.abs(got["direction"] - ref["direction"]).max()) <= 1e-5
        if single is not None:
            one = single(int(sfs[k]), sps[k])
            ok = ok and all((got[key].view(np.uint32) == one[key].view(np.uint32)).all() for key in KEYS)
        if not ok:
            bad.append(int(k))
    return {"rows_checked": [int(k) for k in rows], "mismatching_rows": bad, "ok": not bad,
            "checks": "oracle: dist bit-exact, pred and cutting face exact, direction within 1e-5"
                      + ("; single mnb_cvp: all four outputs bit-exact" if single is not None else "")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3, help="timed calls of each kind (alternated)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--goals", type=int, default=1024)
    ap.add_argument("--size", type=int, default=1000)
    ap.add_argument("--single-sample", type=int, default=64)
    ap.add_argument("--large-size", type=int, default=2236, help="leg 2 grid side (2236 -> 5 M vertices); 0 skips leg 2")
    ap.add_argument("--large-goals", type=int, default=64)
    ap.add_argument("--large-free-gb", type=float, default=12.0, help="leg 2: device memory left free next to the outputs and the ballast")
    args = ap.parse_args()
    import torch
    from oracle import oracle as O
    from mesh_navigation_b200.api import CVPMeshPlanner
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU mode")
    res = {"tool": "gpu_cvp_batch_fields", "gpu": gpu_info()}

    # ---- leg 1: 1 M terrain, 1024 goals, all four outputs vs potentials only ----------------------------------------
    pos, faces, mm, ed, vc, sfs, sps = setup(args.size, args.goals)
    V, n = mm.V, sfs.size
    used0 = used_bytes(torch)
    bufs = outputs(torch, n, V)
    out_bytes = used_bytes(torch) - used0
    mm.use_device_pointers(True)
    used1 = used_bytes(torch)
    fields_call(mm, sfs, sps, bufs)
    ws_bytes = used_bytes(torch) - used1          # the workspace stays allocated after the call
    ws_per_wave = 56 * V + 4 * max(65536, 2 * V)  # ensure_workspace: 64 bytes per vertex on large maps (+ a GroupCtl)
    for _ in range(args.warmup):
        dist_call(mm, sfs, sps, bufs); fields_call(mm, sfs, sps, bufs)
    t_f, t_d, k_f, k_d, st_f, st_d = [], [], [], [], None, None
    for _ in range(args.steps):
        t0 = time.perf_counter(); st_f = fields_call(mm, sfs, sps, bufs); t_f.append(time.perf_counter() - t0); k_f.append(st_f["kernel_ms"])
        t0 = time.perf_counter(); st_d = dist_call(mm, sfs, sps, bufs); t_d.append(time.perf_counter() - t0); k_d.append(st_d["kernel_ms"])
    gpu_during = gpu_info()
    fields_call(mm, sfs, sps, bufs)               # leave the rows of the fields call in the buffers for the parity check
    pf, pd = float(np.mean(t_f)), float(np.mean(t_d))
    res["batch_fields_1m"] = {"mesh_vertices": int(V), "goals": int(n), "outputs": "dist + pred + direction + cutting face, device pointers",
                              "plans_per_s": n / pf, "s_per_call": pf, "kernel_ms_mean": float(np.mean(k_f)), "kernel_ms_min": float(np.min(k_f)),
                              "rounds_summed_over_wavefronts": int(st_f["rounds"]), "settled": int(st_f["settled"]),
                              "deep_labels": int(st_f["deep_labels"]), "steps": args.steps, "warmup": args.warmup}
    res["batch_dist_only_1m"] = {"outputs": "dist, mnb_cvp_batch, device pointers", "plans_per_s": n / pd, "s_per_call": pd,
                                 "kernel_ms_mean": float(np.mean(k_d)), "kernel_ms_min": float(np.min(k_d)),
                                 "note": "alternated call by call with the fields call in the same process"}
    res["epilogue_overhead"] = {"kernel_ms": float(np.mean(k_f) - np.mean(k_d)),
                                "fraction_of_dist_only_kernel_time": float(np.mean(k_f) / np.mean(k_d) - 1.0)}
    res["memory_1m"] = {"output_bytes": int(out_bytes), "workspace_bytes_from_device_memory_growth": int(ws_bytes),
                        "wavefronts_in_flight_from_workspace": int(ws_bytes // ws_per_wave),
                        "device_memory_in_use_bytes": int(used_bytes(torch))}
    # the same goals as single full-field mnb_cvp calls (whole-grid kernel + epilogue), timed on a sample and extrapolated
    one = {k: torch.empty(V, dtype=torch.float32 if k in ("dist", "direction") else torch.int32, device="cuda") for k in KEYS}
    m = min(args.single_sample, n)
    for k in range(2):
        mm.cvp_dev(int(sfs[k]), sps[k], -1, 1.0, 0.3, *[one[key].data_ptr() for key in KEYS])
    single_k = []
    t0 = time.perf_counter()
    for k in range(m):
        mm.cvp_dev(int(sfs[k]), sps[k], -1, 1.0, 0.3, *[one[key].data_ptr() for key in KEYS])
        single_k.append(mm.stats()["kernel_ms"])
    t_single = (time.perf_counter() - t0) / m
    res["single_loop_1m"] = {"sampled_goals": int(m), "ms_per_plan": 1e3 * t_single, "kernel_ms_per_plan": float(np.mean(single_k)),
                             "plans_per_s": 1.0 / t_single, "extrapolated_s_for_all_goals": t_single * n,
                             "note": "loop of full-field mnb_cvp(goal, -1) with all four outputs on a sample of the goals, "
                                     "extrapolated to the whole set (not measured on all of them)"}
    res["batch_fields_vs_single_loop"] = res["batch_fields_1m"]["plans_per_s"] / res["single_loop_1m"]["plans_per_s"]
    mm.use_device_pointers(False)
    pl = CVPMeshPlanner(mm)
    om = O.OracleMesh(pos, faces)
    rows = np.unique(np.linspace(0, n - 1, 8).astype(np.int64))
    res["parity_1m"] = parity(om, ed, vc, sfs, sps, rows, bufs, single=lambda f, p: pl.waveFrontPropagation(f, p))
    mm.close(); del bufs, one, om
    torch.cuda.empty_cache()

    # ---- leg 2: 5 M terrain, 64 goals, all four outputs, with the memory cap binding ---------------------------------
    if args.large_size > 0:
        pos, faces, mm, ed, vc, sfs, sps = setup(args.large_size, args.large_goals)
        V, n = mm.V, sfs.size
        bufs = outputs(torch, n, V)
        free, total = torch.cuda.mem_get_info()
        ballast_bytes = max(0, int(free - args.large_free_gb * 2**30))
        ballast = torch.empty(ballast_bytes, dtype=torch.uint8, device="cuda")
        mm.use_device_pointers(True)
        used0 = used_bytes(torch)
        t0 = time.perf_counter()
        st = fields_call(mm, sfs, sps, bufs)
        t1 = time.perf_counter() - t0
        ws = used_bytes(torch) - used0
        ws_per_wave = 56 * V + 4 * max(65536, 2 * V)
        leg = {"mesh_vertices": int(V), "goals": int(n), "outputs": "dist + pred + direction + cutting face, device pointers",
               "ballast_bytes": ballast_bytes, "free_bytes_before_call": int(total - used0),
               "workspace_bytes_from_device_memory_growth": int(ws), "wavefronts_in_flight_from_workspace": int(ws // ws_per_wave),
               "wavefronts_without_the_cap": "min(goals, CTA slots) = min(%d, SMs x 4)" % n,
               "s_per_call": t1, "kernel_ms": st["kernel_ms"], "plans_per_s": n / t1,
               "device_memory_in_use_bytes": int(used_bytes(torch))}
        mm.use_device_pointers(False)
        del ballast
        om = O.OracleMesh(pos, faces)
        leg["parity"] = parity(om, ed, vc, sfs, sps, [0, n - 1], bufs)
        res["batch_fields_5m_memory_capped"] = leg
        mm.close()
    res["gpu_after_timing"] = gpu_during
    res["parity_ok"] = bool(res["parity_1m"]["ok"] and res.get("batch_fields_5m_memory_capped", {}).get("parity", {"ok": True})["ok"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
