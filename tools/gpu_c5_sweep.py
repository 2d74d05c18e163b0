"""Dev script (GPU box): band-width sweep of the single-plan kernels on a large terrain (config 5: 5000 -> 25 M vertices).
  python tools/gpu_c5_sweep.py [grid side] [comma list of band widths in mean edge weights]"""
import sys, zlib
import numpy as np
sys.path.insert(0, '.')
from mesh_navigation_b200 import synth
from mesh_navigation_b200.api import MeshMap, CVPMeshPlanner, DijkstraMeshPlanner
n = int(sys.argv[1]) if len(sys.argv) > 1 else 5000
ks = [float(x) for x in (sys.argv[2] if len(sys.argv) > 2 else "0,6,10,14,28").split(",")]
pos, faces = synth.grid_mesh(n, n, terrain=True)
mm = MeshMap(pos, faces)
ed = mm.edgeDistances(); mm.setCosts(np.zeros(mm.V, np.float32), ed)
w = float(ed.mean())
c = synth.nearest_vertex(pos, [n * 0.05, n * 0.05, float(pos[:, 2].mean())])
sf = int(2 * ((c // n) * (n - 1) + (c % n))); sp = pos[faces[sf]].mean(0).astype(np.float32)
del pos
for k in ks:
    if k > 0: mm.set_tuning(k * w, 0, 0)
    best = 1e9
    for rep in range(2):
        g = CVPMeshPlanner(mm).waveFrontPropagation(sf, sp); best = min(best, g["kernel_ms"])
    print(f"[{n}x{n}] cvp band {k if k > 0 else 'default (20)'} w: kernel {best:.1f} ms rounds {g['rounds']} evals/V {g['recomputes']/mm.V:.2f} crc {zlib.crc32(g['dist'].tobytes()):08x}", flush=True)
    del g
    best = 1e9
    for rep in range(2):
        d = DijkstraMeshPlanner(mm).dijkstra(int(c)); best = min(best, d["kernel_ms"])
    print(f"[{n}x{n}] dijkstra band {k if k > 0 else 'default (25)'} w: kernel {best:.1f} ms rounds {d['rounds']}", flush=True)
    del d
mm.close()
