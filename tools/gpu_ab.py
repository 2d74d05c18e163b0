"""Dev script (GPU box): A/B of the opt-in variants written without GPU access (round 1), one call, ~2 GPU-minutes.
  python tools/gpu_ab.py [grid side of the single-plan mesh, default 2240]
Prints, for each variant, kernel time + the bit-equality against the default kernel:
  * in-round sweeps / band width of the whole-grid single CVP plan (5 M), band width of the per-CTA batch (1 M, 2 goals
    per SM = one wave)
  * k_layers<true> (shared-memory seen-set) on the 5 M mesh
  * the dynamic-obstacle cycle (inflation update, vector field, incremental layerChanged vs full re-install)"""
import ctypes as C, sys, time
import numpy as np
sys.path.insert(0, '.')
import torch
from mesh_navigation_b200 import synth
from mesh_navigation_b200.api import MeshMap, CVPMeshPlanner, InflationLayer

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2240
pos, faces = synth.grid_mesh(n, n, terrain=True)
mm = MeshMap(pos, faces); ed = mm.edgeDistances(); vc = np.zeros(mm.V, np.float32); mm.setCosts(vc, ed)
mm.L.mnb_debug_set_layers_smem.argtypes = [C.c_void_p, C.c_int32]
c = synth.nearest_vertex(pos, [n * 0.05, n * 0.05, float(pos[:, 2].mean())])
sf = int(2 * ((c // n) * (n - 1) + (c % n))); sp = pos[faces[sf]].mean(0).astype(np.float32)
pl = CVPMeshPlanner(mm)
ref = pl.waveFrontPropagation(sf, sp)['dist'].copy()
# band width / in-round sweeps were tuned (1.8 m / 15) before the causal collapse made an evaluation cheaper: re-scan
mm.L.mnb_debug_set_sweeps.argtypes = [C.c_void_p, C.c_int32]
for (k, delta) in ((15, 1.8), (10, 1.2), (20, 2.4), (30, 3.6), (24, 1.8), (8, 1.8), (0, 0.3)):
    mm.L.mnb_debug_set_sweeps(mm._ctx, k); mm.set_tuning(delta, 0, 0)
    best = 1e9
    for it in range(2):
        g = pl.waveFrontPropagation(sf, sp); best = min(best, g['kernel_ms'])
    print(f"[single {n}x{n}] sweeps={k} delta={delta}: kernel {best:.2f} ms rounds {g['rounds']} recomputes/V {g['recomputes']/mm.V:.2f} "
          f"dist!=default {int((g['dist'].view(np.uint32) != ref.view(np.uint32)).sum())}", flush=True)
mm.L.mnb_debug_set_sweeps(mm._ctx, -1); mm.set_tuning(1.8, 0, 0)
for smem in (0, 1, 0, 1):
    mm.L.mnb_debug_set_layers_smem(mm._ctx, smem)
    for it in range(2):
        Ly = mm.computeLayers()
    if smem == 0: base = Ly
    same = all((Ly[k].view(np.uint32) == base[k].view(np.uint32)).all() for k in ("height_diff", "roughness", "ridge", "combined"))
    print(f"[layers {n}x{n}] smem={smem}: kernel {Ly['kernel_ms']:.2f} ms, identical to default: {same}", flush=True)
mm.L.mnb_debug_set_layers_smem(mm._ctx, 0)
# dynamic-obstacle cycle
infl = InflationLayer(mm)
static = base["combined"]; stat_le = np.where(base["lethal_mask"] != 0)[0]
le0 = np.union1d(stat_le, synth.disc_lethals_grid(pos, n, n, 1000, 0.3, seed=7)).astype(np.uint32)
le1 = np.union1d(stat_le, synth.disc_lethals_grid(pos, n, n, 1000, 0.3, seed=8)).astype(np.uint32)
r0 = infl.onInputChanged(le0)
final = np.maximum(static, np.nan_to_num(r0["cost"], nan=0.0)).astype(np.float32)
mm.computeEdgeWeights(final, 1.0, want_output=False)
t = time.perf_counter(); r1 = infl.onInputChanged(le1); t_infl = time.perf_counter() - t
t = time.perf_counter(); field = infl.vectorMap(); t_vec = time.perf_counter() - t; vec_ms = mm.stats()["kernel_ms"]
ch = r1["changed"]
mm.maxCombinationUpdate([static, r1["cost"]], [0.0, 0.0], None, ch, final, None)
t = time.perf_counter(); mm.layerChanged(ch, final[ch], 1.0); t_inc = time.perf_counter() - t; inc_ms = mm.stats()["kernel_ms"]
gvc, gw = mm.costs()
t = time.perf_counter(); fw = mm.computeEdgeWeights(final, 1.0); t_full = time.perf_counter() - t
print(f"[dynamic {n}x{n}] lethals {le1.size} changed {ch.size}: inflation update {1e3*t_infl:.1f} ms wall ({r1['kernel_ms']:.2f} ms kernels), "
      f"vector field {1e3*t_vec:.1f} ms wall ({vec_ms:.2f} ms kernels), layerChanged incremental {1e3*t_inc:.2f} ms wall ({inc_ms:.3f} ms kernels) "
      f"vs full re-install {1e3*t_full:.1f} ms wall; identical: {bool((gw.view(np.uint32) == fw.view(np.uint32)).all())}", flush=True)
mm.close()
# batch: one wave of goals on the 1M mesh
nb = 1000
bpos, bfaces = synth.grid_mesh(nb, nb, terrain=True)
bm = MeshMap(bpos, bfaces); bm.setCosts(np.zeros(bm.V, np.float32), bm.edgeDistances())
G = 2 * torch.cuda.get_device_properties(0).multi_processor_count     # one wave: 2 CTAs per SM
goals = synth.batch_goal_vertices(bm.V, G, seed=1234)
gi, gj = np.minimum(goals % nb, nb - 2), np.minimum(goals // nb, nb - 2)
sfs = (2 * (gj * (nb - 1) + gi)).astype(np.uint32); sps = bpos[bfaces[sfs]].mean(1).astype(np.float32)
out = torch.empty((G, bm.V), dtype=torch.float32, device='cuda')
for delta in (0.2, 0.3, 0.45, 0.6):
    bm.set_tuning(delta, 1, 0)
    bm.use_device_pointers(True)
    for rep in range(2):
        t = time.perf_counter(); bm.cvp_batch_dev(sfs, sps, 1.0, out.data_ptr()); torch.cuda.synchronize(); dt = time.perf_counter() - t
    bm.use_device_pointers(False)
    st = bm.stats()
    print(f"[batch {G} x 1M] delta={delta}: {1e3*dt:.1f} ms -> {G/dt:.1f} plans/s, recomputes/V {st['recomputes']/G/bm.V:.2f} rounds/plan {st['rounds']/G:.0f}", flush=True)
bm.close()
