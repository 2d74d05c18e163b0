"""Dev script (no GPU): bit-parity of the whole-grid CVP kernel vs the oracle on a LARGE mesh, run on the CPU interpreter
of the kernels (tests/emu).  `python tools/emu_big_parity.py 3200` = 10.24 M vertices: ~2 min map build, ~3 min wavefront
with MNB_EMU_SMS=8, ~25 GB of RAM.  This is the case that exposed the exact-key-tie ordering defect (4 potentials off by
1 ulp, on the GPU and on the interpreter alike) and that verifies its fix (0 mismatches)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("MNB_EMU_SMS", "8")
from tests.emu.run_suite import build
from mesh_navigation_b200 import _lib
_lib.LIB_PATH = build()
import numpy as np
from oracle import oracle as O
from mesh_navigation_b200 import synth
from mesh_navigation_b200.api import MeshMap, CVPMeshPlanner
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
pos, faces = synth.grid_mesh(n, n, terrain=True)
t = time.time(); mm = MeshMap(pos, faces); ed = mm.edgeDistances(); vc = np.zeros(mm.V, np.float32); mm.setCosts(vc, ed)
print(f"map build {time.time() - t:.1f} s", flush=True)
c = synth.nearest_vertex(pos, [n * 0.05, n * 0.05, float(pos[:, 2].mean())])
sf = int(2 * ((c // n) * (n - 1) + (c % n))); sp = pos[faces[sf]].mean(0).astype(np.float32)
om = O.OracleMesh(pos, faces); r = om.cvp(ed, vc, sf, sp); print(f"oracle {r['seconds']:.1f} s", flush=True)
t = time.time(); g = CVPMeshPlanner(mm).waveFrontPropagation(sf, sp); print(f"interpreted k_cvp_grid {time.time() - t:.1f} s, rounds {g['rounds']}", flush=True)
bad = np.where(g['dist'].view(np.uint32) != r['dist'].view(np.uint32))[0]
rel = np.abs(g['dist'][bad].astype(np.float64) - r['dist'][bad]) / r['dist'][bad]
d = r['dist'][np.isfinite(r['dist'])]
print(f"V={mm.V}: dist!= {bad.size} idx {bad[:8].tolist()} maxrel {rel.max() if bad.size else 0:.3e} pred!= {(g['pred'] != r['pred']).sum()} "
      f"backsteps {r['backsteps']} exact key collisions {d.size - np.unique(d).size}", flush=True)
