"""Dev script (no GPU): randomised differential test of the interpreted kernels against the oracle -- random mesh kind /
size / jitter, cost fields, edge_cost_factor, invalid vertices, goal cutoff, cluster sizes, lethal sets, inflation radii.
  python tools/emu_fuzz.py [n_cases] [seed]"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("MNB_EMU_SMS", "4")
from tests.emu.run_suite import build
from mesh_navigation_b200 import _lib
_lib.LIB_PATH = build()
import numpy as np
from oracle import oracle as O
from mesh_navigation_b200 import synth, api
from tests.util import delaunay_mesh, disc_lethals

N = int(sys.argv[1]) if len(sys.argv) > 1 else 20
rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 0)
ONLY = int(sys.argv[3]) if len(sys.argv) > 3 else -1      # replay a single case of the stream
bad = 0
for case in range(N):
    crng = np.random.default_rng(rng.integers(1 << 62))
    if ONLY >= 0 and case != ONLY:
        continue
    kind = crng.choice(["grid", "grid", "planar", "nojitter", "delaunay"])
    if kind == "delaunay":
        pos, faces = delaunay_mesh(int(crng.integers(800, 4000)), seed=int(crng.integers(1 << 30)), with_hub=bool(crng.integers(2)))
    else:
        n = int(crng.integers(24, int(os.environ.get("FUZZ_MAX_N", "140"))))
        pos, faces = synth.grid_mesh(n, n, terrain=kind == "grid", seed=int(crng.integers(1 << 30)), jitter=0.0 if kind == "nojitter" else 0.2)
    om = O.OracleMesh(pos, faces); mm = api.MeshMap(pos, faces); V = om.V
    ed = om.edge_distances()
    cm = crng.integers(3)
    vc = np.zeros(V, np.float32) if cm == 0 else ((crng.random(V) * crng.choice([0.5, 0.9, 1.3])).astype(np.float32) if cm == 1 else
                                                  (np.round(crng.random(V) * 4) / 4 * 0.8).astype(np.float32))
    factor = float(crng.choice([0.0, 1.0, 2.5])) if cm else 0.0
    inv = (crng.random(V) < 0.01).astype(np.uint8) if crng.integers(3) == 0 else None
    w = om.edge_weights(vc, ed, factor)
    mm.setCosts(vc, w, inv)
    sf = int(crng.integers(om.F)); sp = pos[faces[sf]].mean(0).astype(np.float32)
    rf = int(crng.integers(om.F)) if crng.integers(3) == 0 else -1
    cl = float(crng.choice([1.0, 0.8, 5.0]))
    cluster = int(crng.choice([-1, -1, 1, 2, 4]))
    mm.set_tuning(float(crng.choice([0.3, 0.1, 1.8])) if cluster != -1 else 0.0, cluster, 0)
    msg = []
    ref = om.cvp(w, vc, sf, sp, rf, invalid=inv, cost_limit=cl)
    got = api.CVPMeshPlanner(mm, cost_limit=cl).waveFrontPropagation(sf, sp, rf)
    if got["outcome"] != ref["outcome"] or (got["dist"].view(np.uint32) != ref["dist"].view(np.uint32)).any() or (got["pred"] != ref["pred"]).any() \
            or (got["cutting_face"] != ref["cutting_face"]).any() or (got["direction"].view(np.uint32) != ref["direction"].view(np.uint32)).any():
        msg.append(f"CVP outcome {got['outcome']}/{ref['outcome']} dist!= {(got['dist'].view(np.uint32) != ref['dist'].view(np.uint32)).sum()} pred!= {(got['pred'] != ref['pred']).sum()} "
                   f"cut!= {(got['cutting_face'] != ref['cutting_face']).sum()} at {np.where(got['cutting_face'] != ref['cutting_face'])[0][:4].tolist()}")
    # the lean batch round loop (k_cvp_batch): three goals, random cluster size / band width
    bsf = np.concatenate([[sf], crng.integers(0, om.F, 2)]).astype(np.uint32)
    bsp = np.stack([pos[faces[f]].mean(0) for f in bsf]).astype(np.float32); bsp[0] = sp
    bcl = int(crng.choice([1, 1, 2, 4])); mm.set_tuning(float(crng.choice([0.3, 0.1, 0.6])), bcl, 0)
    gb = api.CVPMeshPlanner(mm, cost_limit=cl).waveFrontPropagationBatch(bsf, bsp)
    for i in range(3):
        rb = ref["dist"] if (i == 0 and rf < 0) else om.cvp(w, vc, int(bsf[i]), bsp[i], invalid=inv, cost_limit=cl)["dist"]
        if (gb["dist"][i].view(np.uint32) != rb.view(np.uint32)).any():
            msg.append(f"batch[{i}] cluster {bcl} dist!= {(gb['dist'][i].view(np.uint32) != rb.view(np.uint32)).sum()}")
    mm.set_tuning(0.3, cluster if cluster != -1 else -1, 0)
    sv = int(faces[sf][0]); rv = int(faces[rf][0]) if rf >= 0 else -1
    refd = om.dijkstra(w, vc, sv, rv, invalid=inv, cost_limit=cl)
    gotd = api.DijkstraMeshPlanner(mm, cost_limit=cl).dijkstra(sv, rv)
    if gotd["outcome"] != refd["outcome"] or (gotd["dist"].view(np.uint32) != refd["dist"].view(np.uint32)).any() or (gotd["pred"] != refd["pred"]).any():
        msg.append(f"Dijkstra outcome {gotd['outcome']}/{refd['outcome']} dist!= {(gotd['dist'].view(np.uint32) != refd['dist'].view(np.uint32)).sum()}")
    le = disc_lethals(pos, int(crng.integers(1, 8)), float(crng.choice([0.15, 0.3])), seed=int(crng.integers(1 << 30)))
    rad = float(crng.choice([0.4, 0.7, 1.1]))
    refi = om.inflation(ed, le, invalid=inv, inflation_radius=rad, with_vectors=True)
    il = api.InflationLayer(mm, inflation_radius=rad)
    goti = il.waveCostInflation(le, inv); vec = il.vectorMap()
    if (goti["dist"].view(np.uint32) != refi["dist"].view(np.uint32)).any() or (vec.view(np.uint32) != refi["vectors"].view(np.uint32)).any():
        msg.append(f"inflation dist!= {(goti['dist'].view(np.uint32) != refi['dist'].view(np.uint32)).sum()} vec!= {(vec.view(np.uint32) != refi['vectors'].view(np.uint32)).any(1).sum()}")
    print(f"case {case}: {kind} V={V} costs={cm} factor={factor} invalid={inv is not None} robot={rf >= 0} cluster={cluster} cl={cl} radius={rad} lethals={le.size}: "
          + ("ok" if not msg else "MISMATCH " + "; ".join(msg)), flush=True)
    bad += bool(msg)
    if msg and os.environ.get("FUZZ_DUMP"):      # keep the failing case as a fixture (tests/golden/fuzz_*.npz layout)
        np.savez_compressed(os.path.join(os.environ["FUZZ_DUMP"], f"fuzz_case_{sys.argv[2] if len(sys.argv) > 2 else 0}_{case}.npz"), pos=pos, faces=faces, vc=vc, w=w,
                            inv=inv if inv is not None else np.zeros(0, np.uint8), sf=sf, sp=sp, rf=rf, cl=cl, le=le, rad=rad)
    mm.close()
print(f"{N - bad}/{N} cases bit-identical")
sys.exit(1 if bad else 0)
