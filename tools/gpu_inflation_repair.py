"""Measures the inflation repair (mnb_inflation_repair) against a full mnb_inflation_update on the GPU and prints one JSON
line.

Two contexts hold the same map: one runs repairs, the other full updates, alternated call by call on the same lethal
sets, all with device pointers (torch tensors).  Every call's distances, riskiness and changed set are checked: the
repair's against the full call's bit for bit, and the changed set against the bitwise diff of consecutive full results.
The map is the bench's 5 M-vertex terrain (2240 x 2240) with its layer lethals (mnb_compute_layers) plus the bench's
1000 obstacle discs of 0.3 m.  Each workload switches between two lethal sets A and B (A -> B -> A ...), first once
untimed.  Times: the host clock around each call (the library synchronises before it returns) and the CUDA-event time
the library reports; medians over the timed calls.
Workloads:
  one_disc:    one disc moves 0.2 m
  ten_discs:   10 discs move 0.2 m
  100_discs, 334_discs: every 10th / every 3rd disc moves 0.2 m
  touch_layer: one disc moves next to a layer-lethal vertex
  all_discs:   all 1000 discs move (the bench's seeds 7 and 8)
Each workload also reports the affected share the call bases its choice of the whole-map wave on (the old footprint's
vertices in clusters that contain or share a face with a changed lethal, over the old footprint), computed here in
numpy from the full call's distances.
Chain (1 M terrain, 256 Dijkstra rows): after a disc move, mnb_dijkstra_batch_repair with the full call's update set
against the same repair with the repair's changed set; both repaired row sets are checked bit for bit against a fresh
mnb_dijkstra_batch.
Usage: python tools/gpu_inflation_repair.py [--reps N] [--out FILE]"""
import argparse
import ctypes as C
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


def disc_at(pos, n, centre, radius=0.3, h=0.1):
    """vertices within radius (xy) of vertex `centre` of an n x n grid_mesh"""
    k = int(np.ceil(radius / h)) + 2
    ci, cj = centre % n, centre // n
    ii, jj = np.meshgrid(np.arange(max(0, ci - k), min(n, ci + k + 1)), np.arange(max(0, cj - k), min(n, cj + k + 1)))
    idx = (jj * n + ii).ravel()
    d = pos[idx, :2] - pos[centre, :2]
    return idx[(d ** 2).sum(1) <= radius * radius]


def affected_share(faces, dist, old_le, new_le):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    V = dist.size
    foot = np.isfinite(dist)
    f = faces.astype(np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [0, 2]]])
    e = e[foot[e[:, 0]] & foot[e[:, 1]]]
    _, comp = connected_components(coo_matrix((np.ones(len(e), np.int8), (e[:, 0], e[:, 1])), shape=(V, V)), directed=False)
    delta = np.zeros(V, bool)
    delta[np.setxor1d(old_le, new_le)] = True
    touched = np.zeros(V, bool)
    touched[faces[delta[faces].any(1)].ravel()] = True
    touched |= delta
    hit = np.zeros(comp.max() + 1, bool)
    hit[comp[touched & foot]] = True
    return float(hit[comp[foot]].mean())


def changed_of(new, old):
    diff = (new.view(np.uint32) != old.view(np.uint32)) & ~(np.isnan(new) & np.isnan(old))
    return np.where(diff)[0].astype(np.uint32)


class Pair:
    def __init__(self, torch, pos, faces):
        from mesh_navigation_b200.api import InflationLayer, MeshMap
        self.torch = torch
        self.maps = [MeshMap(pos, faces), MeshMap(pos, faces)]          # [0] repair, [1] full update
        self.V = self.maps[0].V
        self.layers = [InflationLayer(m) for m in self.maps]
        for m in self.maps:
            m.use_device_pointers(True)
        t = lambda dt: torch.empty(self.V, dtype=dt, device="cuda")
        self.out = [(t(torch.float32), t(torch.float32), t(torch.int32)) for _ in range(2)]
        self.prev = None

    def call(self, k, le_dev, n):
        m, (d, c, ch) = self.maps[k], self.out[k]
        fn = m.L.mnb_inflation_repair if k == 0 else m.L.mnb_inflation_update
        cnt = C.c_uint32(0)
        t0 = time.perf_counter()
        m._check(fn(m._ctx, C.c_void_p(le_dev.data_ptr()), n, None, C.byref(self.layers[k].config), C.c_void_p(d.data_ptr()),
                    C.c_void_p(c.data_ptr()), C.c_void_p(ch.data_ptr()), C.byref(cnt)))
        wall = (time.perf_counter() - t0) * 1e3
        return dict(wall_ms=wall, n=cnt.value, **m.stats())

    def step(self, le):
        torch = self.torch
        le_dev = torch.from_numpy(le.view(np.int32)).cuda()
        torch.cuda.synchronize()
        r = self.call(0, le_dev, le.size)
        f = self.call(1, le_dev, le.size)
        rd, rc, rch = [x.cpu().numpy() for x in self.out[0]]
        fd, fc, fch = [x.cpu().numpy() for x in self.out[1]]
        ok = bool((rd.view(np.uint32) == fd.view(np.uint32)).all() and (rc.view(np.uint32) == fc.view(np.uint32)).all())
        if self.prev is not None:
            ok = ok and bool(np.array_equal(rch[:r["n"]].view(np.uint32), changed_of(fc, self.prev)))
        self.prev = fc
        return r, f, ok, rch[:r["n"]].view(np.uint32).copy(), fch[:f["n"]].view(np.uint32).copy()

    def close(self):
        for m in self.maps:
            m.use_device_pointers(False)
            m.close()


def run_workload(pair, faces, a, b, reps):
    pair.step(a); pair.step(b); pair.step(a)                          # warm-up (and the first repair builds the cluster ids)
    share = affected_share(faces, pair.out[1][0].cpu().numpy(), a, b)
    rec = []
    for i in range(reps):
        r, f, ok, rch, fch = pair.step(b if i % 2 == 0 else a)
        rec.append(dict(ok=ok, rep_wall=r["wall_ms"], rep_kernel=r["kernel_ms"], full_wall=f["wall_ms"], full_kernel=f["kernel_ms"],
                        rounds=r["rounds"], full_rounds=f["rounds"], settled=r["settled"], full_settled=f["settled"],
                        launches=r["kernel_launches"], changed=int(rch.size), update_set=int(fch.size)))
    med = lambda k: float(np.median([x[k] for x in rec]))
    return dict(ok=all(x["ok"] for x in rec), affected_share=share, repair_wall_ms=med("rep_wall"), repair_kernel_ms=med("rep_kernel"),
                full_wall_ms=med("full_wall"), full_kernel_ms=med("full_kernel"), rounds=med("rounds"), full_rounds=med("full_rounds"),
                settled=med("settled"), full_settled=med("full_settled"), launches=med("launches"),
                changed=med("changed"), update_set=med("update_set"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from mesh_navigation_b200 import synth
    from mesh_navigation_b200.api import DijkstraMeshPlanner, InflationLayer, MeshMap
    res = {"gpu": gpu_info()}
    n = 2240
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=42)
    mm = MeshMap(pos, faces)
    layer = np.where(mm.computeLayers()["lethal_mask"] != 0)[0].astype(np.uint32)
    mm.close()
    V = n * n
    centres = synth.pcg32_stream(7, 1000, V).astype(np.int64)
    discs = [disc_at(pos, n, int(c)) for c in centres]
    lethals = lambda ds: np.unique(np.concatenate([layer] + ds)).astype(np.uint32)
    shift = lambda c: int(c + 2 if (c % n) + 2 < n else c - 2)        # 2 vertices = 0.2 m along x
    A = lethals(discs)
    moved = lambda ks: lethals([disc_at(pos, n, shift(int(centres[k]))) if k in ks else discs[k] for k in range(len(discs))])
    li = int(layer[len(layer) // 2])
    touch = lethals(discs[1:] + [disc_at(pos, n, li + 4 if (li % n) + 4 < n else li - 4)])
    B_all = np.union1d(layer, synth.disc_lethals_grid(pos, n, n, 1000, 0.3, seed=8)).astype(np.uint32)
    pair = Pair(torch, pos, faces)
    res["lethal_vertices"] = int(A.size)
    res["one_disc"] = run_workload(pair, faces, A, moved({0}), args.reps)
    res["ten_discs"] = run_workload(pair, faces, A, moved(set(range(0, 1000, 100))), args.reps)
    res["100_discs"] = run_workload(pair, faces, A, moved(set(range(0, 1000, 10))), args.reps)
    res["334_discs"] = run_workload(pair, faces, A, moved(set(range(0, 1000, 3))), args.reps)
    res["touch_layer"] = run_workload(pair, faces, A, touch, args.reps)
    res["all_discs"] = run_workload(pair, faces, np.union1d(layer, synth.disc_lethals_grid(pos, n, n, 1000, 0.3, seed=7)).astype(np.uint32),
                                    B_all, args.reps)
    pair.close()
    # downstream chain on the 1 M map: the Dijkstra field repair fed with the update set or with the changed set
    n1 = 1000
    pos1, faces1 = synth.grid_mesh(n1, n1, terrain=True, seed=42)
    mm = MeshMap(pos1, faces1)
    V1 = mm.V
    mm.computeEdgeWeights(np.zeros(V1, np.float32), 1.0, want_output=False)
    infl = InflationLayer(mm)
    pl = DijkstraMeshPlanner(mm, cost_limit=0.95)
    seeds = synth.batch_goal_vertices(V1, 256, seed=1234).astype(np.uint32)
    c1 = synth.pcg32_stream(7, 199, V1).astype(np.int64)
    d1 = [disc_at(pos1, n1, int(c)) for c in c1]
    base = np.unique(np.concatenate(d1)).astype(np.uint32)
    infl.onInputChanged(base)
    mm.layerChanged(np.arange(V1, dtype=np.uint32), np.zeros(V1, np.float32), 1.0, by_vertex=True)
    old = infl.onInputChanged(base)["cost"]
    rows = [torch.empty((256, V1), dtype=torch.float32, device="cuda"), torch.empty((256, V1), dtype=torch.int32, device="cuda")]
    mm.use_device_pointers(True)
    try:
        mm.dijkstra_batch_dev(seeds, 0.95, rows[0].data_ptr(), rows[1].data_ptr())
    finally:
        mm.use_device_pointers(False)
    le = np.unique(np.concatenate([base, disc_at(pos1, n1, int(c1[0]) + 2)])).astype(np.uint32)
    r = infl.repairInflation(le)
    update_set = np.where(~np.isnan(r["cost"]) | ~np.isnan(old))[0].astype(np.uint32)   # what onInputChanged reports
    mm.layerChanged(r["changed"], r["cost"], 1.0, by_vertex=True, default_value=0.0)
    fresh = [torch.empty_like(rows[0]), torch.empty_like(rows[1])]
    mm.use_device_pointers(True)
    try:
        mm.dijkstra_batch_dev(seeds, 0.95, fresh[0].data_ptr(), fresh[1].data_ptr())
    finally:
        mm.use_device_pointers(False)
    chain = []
    for name, ch in (("update_set", update_set), ("changed_set", r["changed"])):
        d, q = rows[0].clone(), rows[1].clone()
        torch.cuda.synchronize()
        mm.use_device_pointers(True)
        try:
            t0 = time.perf_counter()
            mm.dijkstra_batch_repair_dev(seeds, ch, 0.95, d.data_ptr(), q.data_ptr())
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
        finally:
            mm.use_device_pointers(False)
        st = mm.stats()
        same = bool(torch.equal(d.view(torch.int32), fresh[0].view(torch.int32)) and torch.equal(q, fresh[1]))
        chain.append(dict(input=name, set_size=int(ch.size), wall_ms=wall, kernel_ms=st["kernel_ms"], recomputes=st["recomputes"],
                          rows_equal_fresh_batch=same))
        del d, q
    res["chain_1m_256_rows"] = chain
    mm.close()
    res["ok"] = all(res[k]["ok"] for k in ("one_disc", "ten_discs", "100_discs", "334_discs", "touch_layer", "all_discs")) and \
        all(c["rows_equal_fresh_batch"] for c in chain)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0 if res["ok"] else 1


if __name__ == "__main__":
    sys.exit(main())
