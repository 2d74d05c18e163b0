"""exercise layers + inflation + dijkstra + batch once each (for ncu captures)"""
import sys, numpy as np, torch
sys.path.insert(0,'.')
from mesh_navigation_b200 import synth
from mesh_navigation_b200.api import MeshMap, CVPMeshPlanner, DijkstraMeshPlanner, InflationLayer
from tests.util import disc_lethals
n=int(sys.argv[1])
pos,faces=synth.grid_mesh(n,n,terrain=True)
mm=MeshMap(pos,faces); ed=mm.edgeDistances(); mm.setCosts(np.zeros(mm.V,np.float32), ed)
for rep in range(2):
    L=mm.computeLayers(); print("layers ms", L['kernel_ms'], "lethal", int((L['lethal_mask']!=0).sum()))
    le=np.union1d(np.where(L['lethal_mask']!=0)[0], disc_lethals(pos, 1000 if n>=1000 else 20, 0.3)).astype(np.uint32)
    I=InflationLayer(mm).waveCostInflation(le); print("inflate ms", I['kernel_ms'], "rounds", I['rounds'], "labelled", int(np.isfinite(I['dist']).sum()), "recomputes", I['recomputes'])
    D=DijkstraMeshPlanner(mm).dijkstra(n*n//2+n//2); print("dijkstra ms", D['kernel_ms'], "rounds", D['rounds'])
    goals=synth.batch_goal_vertices(mm.V, 2*torch.cuda.get_device_properties(0).multi_processor_count, seed=1234)
    gi,gj=np.minimum(goals%n,n-2), np.minimum(goals//n,n-2)
    sfs=(2*(gj*(n-1)+gi)).astype(np.uint32); sps=pos[faces[sfs]].mean(1).astype(np.float32)
    if len(sys.argv)>2:
        B=CVPMeshPlanner(mm).waveFrontPropagationBatch(sfs[:int(sys.argv[2])], sps[:int(sys.argv[2])]); print("batch ms", B['kernel_ms'])
