"""Measures the batch replan (mnb_cvp_batch_replan) against a fresh mnb_cvp_batch_fields on the GPU and prints one JSON
line.

Every call works on device rows (MNB_PTR_DEVICE, torch tensors), all four outputs.  After each cost update the two calls
alternate on the same updated map: the batch replan into one set of rows, then a fresh batch into a second set, and
every row is compared bit for bit.  Each leg first runs one update -> replan -> batch cycle untimed (warm-up of every
shape).  Times: the host clock around each call (the library synchronises its stream before it returns) and the kernel
time the library reads from CUDA events (the batch kernel; the small T0 launch before it is not in it).  Per call: the
settled share (replan settled / fresh settled) and the resident goals (slots that hold a wave after the call).
Goals: the config-4 goal vertices (synth.batch_goal_vertices(V, n, seed=1234)), the grid face at each, its centroid.
Legs:
  discs_1m_64 / discs_1m_256: the 1 M-vertex terrain, 64 / 256 goals; a 0.3 m disc of cost 0.8 (cost limit 0.95)
             appears at 6 random places, one at a time, and each is removed again.
  moving_1m: the 1 M terrain, 64 goals; the obstacle discs of the bench's dynamic-obstacle cycle (199 discs) move between
             two seeds through InflationLayer.onInputChanged -> layerChanged.  Most of the map changes: the adversarial case.
  discs_5m:  the 5 M-vertex terrain (2240 x 2240), 64 goals, 3 discs appear and are removed again; the slots take what
             device memory the workspace and the two sets of rows leave.
Usage: python tools/gpu_cvp_batch_replan.py [--legs discs_1m_64,discs_1m_256,moving_1m,discs_5m] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COST_LIMIT = 0.95


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except Exception as e:      # reported, not hidden
        return {"error": f"nvidia-smi: {e}"}


class Leg:
    def __init__(self, torch, n, n_goals):
        from mesh_navigation_b200 import synth
        from mesh_navigation_b200.api import InflationLayer, MeshMap
        self.torch, self.n = torch, n
        self.pos, self.faces = synth.grid_mesh(n, n, terrain=True, seed=42)
        self.mm = MeshMap(self.pos, self.faces)
        self.V = self.mm.V
        self.mm.computeEdgeWeights(np.zeros(self.V, np.float32), 1.0, want_output=False)
        goals = synth.batch_goal_vertices(self.V, n_goals, seed=1234)
        gi, gj = np.minimum(goals % n, n - 2), np.minimum(goals // n, n - 2)
        self.sf = (2 * (gj * (n - 1) + gi)).astype(np.uint32)
        self.sp = self.pos[self.faces[self.sf]].mean(1).astype(np.float32)
        self.infl = InflationLayer(self.mm)
        shape = (n_goals, self.V)
        mk = lambda: [torch.empty(shape, dtype=t, device="cuda") for t in (torch.float32, torch.int32, torch.float32, torch.int32)]
        self.rows, self.fresh_rows = mk(), mk()

    def call(self, f):
        self.mm.use_device_pointers(True)
        try:
            t0 = time.perf_counter()
            rc = f()
            self.torch.cuda.synchronize()
            return rc, 1e3 * (time.perf_counter() - t0), self.mm.stats()
        finally:
            self.mm.use_device_pointers(False)

    def replan(self, changed):
        return self.call(lambda: self.mm.cvp_batch_replan_dev(self.sf, self.sp, COST_LIMIT, changed, *[x.data_ptr() for x in self.rows]))

    def fresh(self):
        return self.call(lambda: self.mm.cvp_batch_fields_dev(self.sf, self.sp, COST_LIMIT, *[x.data_ptr() for x in self.fresh_rows]))

    def step(self, changed, timed, rec):
        rc_r, t_r, s_r = self.replan(changed)
        slots = self.mm.batch_replan_slots()
        rc_f, t_f, s_f = self.fresh()
        same = rc_r == rc_f and all(self.torch.equal(a.view(self.torch.int32), b.view(self.torch.int32)) for a, b in zip(self.rows, self.fresh_rows))
        if not same:
            raise SystemExit(json.dumps({"error": "batch replan differs from the fresh batch", "changed": int(len(changed))}))
        if timed:
            rec.append(dict(changed=int(len(changed)), replan_ms=t_r, replan_kernel_ms=s_r["kernel_ms"], batch_ms=t_f,
                            batch_kernel_ms=s_f["kernel_ms"], settled_share=s_r["settled"] / max(1, s_f["settled"]),
                            resident_goals=slots[1], slots=slots[0]))

    def disc(self, centre, radius=0.3):
        d = np.linalg.norm(self.pos[:, :2] - self.pos[centre, :2][None, :], axis=1)
        return np.where(d <= radius)[0].astype(np.uint32)

    def update(self, changed, value):
        self.mm.layerChanged(changed, np.full(changed.size, value, np.float32), 1.0)

    def close(self):
        self.mm.close()


def summary(rec):
    keys = [k for k in rec[0] if k != "changed"]
    out = {k: float(np.median([r[k] for r in rec])) for k in keys}
    out.update(calls=len(rec), changed_median=float(np.median([r["changed"] for r in rec])))
    return out


def leg_discs(torch, n, n_goals, n_discs, seed):
    lg = Leg(torch, n, n_goals)
    rng = np.random.default_rng(seed)
    centres = rng.choice(lg.V, n_discs + 1, replace=False)
    rec = []
    lg.step(np.empty(0, np.uint32), False, rec)
    warm = lg.disc(centres[-1])
    lg.update(warm, 0.8); lg.step(warm, False, rec)
    lg.update(warm, 0.0); lg.step(warm, False, rec)
    discs = [lg.disc(c) for c in centres[:n_discs]]
    for d in discs:
        lg.update(d, 0.8); lg.step(d, True, rec)
    for d in discs:
        lg.update(d, 0.0); lg.step(d, True, rec)
    lg.close()
    return dict(vertices=lg.V, goals=n_goals, appear=summary(rec[:n_discs]), remove=summary(rec[n_discs:]), per_call=rec)


def leg_moving(torch, n, n_goals, cycles):
    from mesh_navigation_b200 import synth
    lg = Leg(torch, n, n_goals)
    n_discs = max(2, int(round(1000 * (n / 2240.0) ** 2)))
    le = [synth.disc_lethals_grid(lg.pos, n, n, n_discs, 0.3, seed=s).astype(np.uint32) for s in (7, 8)]

    def move(k):
        r = lg.infl.onInputChanged(le[k])
        lg.mm.layerChanged(r["changed"], r["cost"], 1.0, by_vertex=True, default_value=0.0)
        return r["changed"]

    rec = []
    move(0)
    lg.step(np.empty(0, np.uint32), False, rec)
    lg.step(move(1), False, rec); lg.step(move(0), False, rec)
    for c in range(cycles):
        lg.step(move(1 - c % 2), True, rec)
    lg.close()
    return dict(vertices=lg.V, goals=n_goals, discs=n_discs, moves=summary(rec), per_call=rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="discs_1m_64,discs_1m_256,moving_1m,discs_5m")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this script measures on the device only")
    res = {"gpu_before": gpu_info()}
    legs = args.legs.split(",")
    if "discs_1m_64" in legs:
        res["discs_1m_64"] = leg_discs(torch, 1000, 64, 6, seed=5)
    if "discs_1m_256" in legs:
        res["discs_1m_256"] = leg_discs(torch, 1000, 256, 6, seed=5)
    if "moving_1m" in legs:
        res["moving_1m"] = leg_moving(torch, 1000, 64, 4)
    if "discs_5m" in legs:
        res["discs_5m"] = leg_discs(torch, 2240, 64, 3, seed=6)
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
