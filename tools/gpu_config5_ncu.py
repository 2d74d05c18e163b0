"""Dev script (GPU box, under ncu): one launch each of the fused layers, the single-plan CVP wavefront and the single-plan
Dijkstra wavefront on the config-5 terrain (5000 x 5000 = 25 M vertices)."""
import sys
import numpy as np
sys.path.insert(0, '.')
from mesh_navigation_b200 import synth
from mesh_navigation_b200.api import MeshMap, CVPMeshPlanner, DijkstraMeshPlanner
n = int(sys.argv[1]) if len(sys.argv) > 1 else 5000
pos, faces = synth.grid_mesh(n, n, terrain=True)
mm = MeshMap(pos, faces)
ed = mm.edgeDistances(); mm.setCosts(np.zeros(mm.V, np.float32), ed)
L = mm.computeLayers(); print("layers", L["kernel_ms"], flush=True); del L
c = synth.nearest_vertex(pos, [n * 0.05, n * 0.05, float(pos[:, 2].mean())])
sf = int(2 * ((c // n) * (n - 1) + (c % n))); sp = pos[faces[sf]].mean(0).astype(np.float32)
g = CVPMeshPlanner(mm).waveFrontPropagation(sf, sp); print("cvp", g["kernel_ms"], g["rounds"], flush=True); del g
d = DijkstraMeshPlanner(mm).dijkstra(int(c)); print("dijkstra", d["kernel_ms"], d["rounds"], flush=True)
mm.close()
