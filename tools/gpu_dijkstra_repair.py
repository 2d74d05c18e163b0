"""Measures the Dijkstra field repair (mnb_dijkstra_batch_repair) against a fresh mnb_dijkstra_batch on the GPU and prints
one JSON line.

Every call works on device rows (MNB_PTR_DEVICE, torch tensors).  After each cost update the two calls are alternated on
the same updated map: the repair of the resident rows, then a fresh batch into a second pair of rows, and every repaired
row is compared with the fresh one bit for bit (distances as uint32, predecessors).  Each leg first runs one update ->
repair -> batch cycle untimed (warm-up of every shape).  Times: the host clock around each call (the library synchronises
its stream before it returns) and the kernel time the library reads from CUDA events.  Per call the script reports ms for
both calls, recomputes per wave and rounds per wave (mnb_get_stats, summed over the waves).
Legs:
  discs_1m:  the 1 M-vertex terrain (synth.grid_mesh(1000, 1000, terrain=True)), 1024 fields at the config-4 goals
             (synth.batch_goal_vertices(V, 1024, seed=1234)), edge_cost_factor 1; a 0.3 m disc of +inf cost appears at 16
             random places, one at a time, then each is removed again.
  moving_1m: the same map and fields; the obstacle discs of the bench's dynamic-obstacle cycle at the bench's density
             (1000 discs on the 5 M map, 199 on the 1 M one) move between two seeds: InflationLayer.onInputChanged ->
             layerChanged(changed, riskiness) -> repair with that changed set.  Most of the map changes here.
  discs_5m:  the 5 M-vertex terrain (2240 x 2240), 256 fields, 4 discs appear and are removed again; the repair and the
             batch run under the batch calls' memory cap.
Usage: python tools/gpu_dijkstra_repair.py [--legs discs_1m,moving_1m,discs_5m] [--out FILE]
(--out: the full result, per-call records included, as one JSON line)"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COST_LIMIT = 0.95      # below the inscribed / lethal values of the inflation, so obstacles do not expand


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except Exception as e:      # reported, not hidden
        return {"error": f"nvidia-smi: {e}"}


class Leg:
    def __init__(self, torch, n, n_fields):
        from mesh_navigation_b200 import synth
        from mesh_navigation_b200.api import DijkstraMeshPlanner, InflationLayer, MeshMap
        self.torch, self.n = torch, n
        self.pos, self.faces = synth.grid_mesh(n, n, terrain=True, seed=42)
        self.mm = MeshMap(self.pos, self.faces)
        self.V = self.mm.V
        self.mm.computeEdgeWeights(np.zeros(self.V, np.float32), 1.0, want_output=False)
        self.seeds = synth.batch_goal_vertices(self.V, n_fields, seed=1234).astype(np.uint32)
        self.infl = InflationLayer(self.mm)
        self.pl = DijkstraMeshPlanner(self.mm, cost_limit=COST_LIMIT)
        shape = (n_fields, self.V)
        self.dist = torch.empty(shape, dtype=torch.float32, device="cuda")
        self.pred = torch.empty(shape, dtype=torch.int32, device="cuda")
        self.fdist = torch.empty(shape, dtype=torch.float32, device="cuda")
        self.fpred = torch.empty(shape, dtype=torch.int32, device="cuda")
        self.mm.use_device_pointers(False)

    def fresh(self, dist, pred):
        self.mm.use_device_pointers(True)
        try:
            t0 = time.perf_counter()
            assert self.mm.dijkstra_batch_dev(self.seeds, COST_LIMIT, dist.data_ptr(), pred.data_ptr()) == 0
            self.torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), self.mm.stats()
        finally:
            self.mm.use_device_pointers(False)

    def repair(self, changed):
        self.mm.use_device_pointers(True)
        try:
            t0 = time.perf_counter()
            assert self.mm.dijkstra_batch_repair_dev(self.seeds, changed, COST_LIMIT, self.dist.data_ptr(), self.pred.data_ptr()) == 0
            self.torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), self.mm.stats()
        finally:
            self.mm.use_device_pointers(False)

    def update(self, changed, values):
        self.mm.layerChanged(np.asarray(changed, np.uint32), np.asarray(values, np.float32), 1.0)

    def step(self, changed, timed, rec):
        """repair, then a fresh batch into the second rows; the repaired rows must equal the fresh ones bit for bit"""
        t_rep, s_rep = self.repair(changed)
        t_fr, s_fr = self.fresh(self.fdist, self.fpred)
        same = bool(self.torch.equal(self.dist.view(self.torch.int32), self.fdist.view(self.torch.int32)) and
                    self.torch.equal(self.pred, self.fpred))
        if not same:
            raise SystemExit(json.dumps({"error": "repaired rows differ from the fresh batch", "changed": int(len(changed))}))
        if timed:
            k = len(self.seeds)
            rec.append(dict(changed=int(len(changed)), repair_ms=t_rep, repair_kernel_ms=s_rep["kernel_ms"],
                            batch_ms=t_fr, batch_kernel_ms=s_fr["kernel_ms"],
                            repair_recomputes_per_wave=s_rep["recomputes"] / k, batch_recomputes_per_wave=s_fr["recomputes"] / k,
                            repair_rounds_per_wave=s_rep["rounds"] / k, batch_rounds_per_wave=s_fr["rounds"] / k))

    def disc(self, centre, radius=0.3):
        d = np.linalg.norm(self.pos[:, :2] - self.pos[centre, :2][None, :], axis=1)
        return np.where(d <= radius)[0].astype(np.uint32)

    def close(self):
        self.mm.close()


def summary(rec):
    keys = [k for k in rec[0] if k != "changed"]
    out = {k: float(np.median([r[k] for r in rec])) for k in keys}
    out.update(calls=len(rec), changed_median=float(np.median([r["changed"] for r in rec])),
               repair_ms_total=float(sum(r["repair_ms"] for r in rec)), batch_ms_total=float(sum(r["batch_ms"] for r in rec)))
    return out


def leg_discs(torch, n, n_fields, n_discs, seed):
    lg = Leg(torch, n, n_fields)
    lg.fresh(lg.dist, lg.pred)
    rng = np.random.default_rng(seed)
    centres = rng.choice(lg.V, n_discs + 1, replace=False)
    rec = []
    warm = lg.disc(centres[-1])
    lg.update(warm, np.full(warm.size, np.inf)); lg.step(warm, False, rec)
    lg.update(warm, np.zeros(warm.size)); lg.step(warm, False, rec)
    discs = [lg.disc(c) for c in centres[:n_discs]]
    for d in discs:                                          # appear, one at a time
        lg.update(d, np.full(d.size, np.inf)); lg.step(d, True, rec)
    for d in discs:                                          # removed again, one at a time
        lg.update(d, np.zeros(d.size)); lg.step(d, True, rec)
    lg.close()
    return dict(vertices=lg.V, fields=n_fields, appear=summary(rec[:n_discs]), remove=summary(rec[n_discs:]), per_call=rec)


def leg_moving(torch, n, n_fields, cycles):
    from mesh_navigation_b200 import synth
    lg = Leg(torch, n, n_fields)
    n_discs = max(2, int(round(1000 * (n / 2240.0) ** 2)))
    le = [synth.disc_lethals_grid(lg.pos, n, n, n_discs, 0.3, seed=s).astype(np.uint32) for s in (7, 8)]

    def move(k):
        r = lg.infl.onInputChanged(le[k])
        lg.mm.layerChanged(r["changed"], r["cost"], 1.0, by_vertex=True, default_value=0.0)
        return r["changed"]

    move(0)
    lg.fresh(lg.dist, lg.pred)
    rec = []
    lg.step(move(1), False, rec); lg.step(move(0), False, rec)
    for c in range(cycles):
        lg.step(move(1 - c % 2), True, rec)
    lg.close()
    return dict(vertices=lg.V, fields=n_fields, discs=n_discs, moves=summary(rec), per_call=rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="discs_1m,moving_1m,discs_5m")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this script measures on the device only")
    res = {"gpu_before": gpu_info()}
    legs = args.legs.split(",")
    if "discs_1m" in legs:
        res["discs_1m"] = leg_discs(torch, 1000, 1024, 16, seed=5)
    if "moving_1m" in legs:
        res["moving_1m"] = leg_moving(torch, 1000, 1024, 4)
    if "discs_5m" in legs:
        res["discs_5m"] = leg_discs(torch, 2240, 256, 4, seed=6)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    short = {k: ({kk: vv for kk, vv in v.items() if kk != "per_call"} if isinstance(v, dict) else v) for k, v in res.items()}
    print(json.dumps(short))


if __name__ == "__main__":
    main()
