"""Who owns the device memory of the host layer (csrc/meshnav.cu, csrc/raycast_host.cuh), on the CPU interpreter (no GPU).

The interpreter's cudaMalloc refuses a single request above MNB_EMU_MALLOC_LIMIT bytes, and mnb_emu_allocated_bytes()
reports what is allocated and not freed (tests/emu/cuda_runtime.h).  With the two, the allocation-failure paths of the
entry points can be walked: a buffer that failed to grow must not keep the capacity of the one it replaced, an error
return must release what the call had allocated, and a mesh change or mnb_destroy must release everything they own.
Every scenario runs in a process of its own (python tests/test_emu_host_memory.py <scenario>), so that a write through a
null pointer is a failed assertion here and not the end of the test run.  Nothing here runs on a real device."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_LIB = os.path.join(ROOT, "tests", "emu", "libmeshnav_emu.so")
PAGE = 4096                 # the interpreter rounds every allocation up to whole pages
MNB_E_CUDA = -2


# ---- scenarios (run in the child process) ------------------------------------------------------------------------------
def limit(n_bytes=None):
    if n_bytes is None:
        os.environ.pop("MNB_EMU_MALLOC_LIMIT", None)
    else:
        os.environ["MNB_EMU_MALLOC_LIMIT"] = str(n_bytes)


def allocated(L):
    L.mnb_emu_allocated_bytes.restype = C.c_size_t
    return L.mnb_emu_allocated_bytes()


def fails_with_cuda_error(A, call):
    with pytest.raises(A.MeshNavError, match=f"error {MNB_E_CUDA}:"):
        call()


def planning_map(A, n=12):
    from mesh_navigation_b200 import synth
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=3)
    mm = A.MeshMap(pos, faces)
    mm.setCosts(np.zeros(mm.V, np.float32), mm.edgeDistances())
    return mm, pos, faces


def seeds_of(pos, faces, n):
    sf = (np.arange(n, dtype=np.uint32) * 7) % faces.shape[0]
    return sf, pos[faces[sf]].mean(1).astype(np.float32)


def same_bits(a, b):
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def stale_seed_capacity(A, O):
    mm, pos, faces = planning_map(A)
    cvp = A.CVPMeshPlanner(mm)
    first = cvp.waveFrontPropagationBatch(*seeds_of(pos, faces, 2))["dist"]
    limit(4000)             # the seed faces of 2000 goals are 8000 bytes
    fails_with_cuda_error(A, lambda: cvp.waveFrontPropagationBatch(*seeds_of(pos, faces, 2000)))
    limit()
    assert same_bits(cvp.waveFrontPropagationBatch(*seeds_of(pos, faces, 2))["dist"], first)
    mm.close()


def stale_ray_staging_capacity(A, O):
    mm, pos, faces = planning_map(A)
    rng = np.random.default_rng(5)
    o = (pos.min(0) + rng.random((5000, 3)) * (pos.max(0) - pos.min(0)) + [0, 0, 1]).astype(np.float32)
    down = np.array([0, 0, -1], np.float32)
    first = mm.castRays(o[:8], down)
    limit(1000)             # the staged origins and direction of 5000 rays are 60 kB
    fails_with_cuda_error(A, lambda: mm.castRays(o, down))
    limit()
    again, ref = mm.castRays(o[:8], down), O.OracleMesh(pos, faces).cast_rays(o[:8], down)
    for k in ("hit", "face"):
        assert (again[k] == first[k]).all() and (again[k] == ref[k]).all()
    for k in ("dist", "point"):
        assert same_bits(again[k], first[k]) and same_bits(again[k], ref[k])
    mm.close()


def stale_output_capacity(A, O):
    mm, pos, faces = planning_map(A)
    dij = A.DijkstraMeshPlanner(mm)
    first = dij.dijkstraBatch([17])
    limit(50000)            # the seeds of 300 waves fit, their 300 x V distance rows (172 kB) do not
    fails_with_cuda_error(A, lambda: dij.dijkstraBatch(np.arange(300) % mm.V))
    limit()
    again = dij.dijkstraBatch([17])
    assert same_bits(again["dist"], first["dist"]) and (again["pred"] == first["pred"]).all()
    mm.close()


def no_leak_on_error_return(A, O):
    mm, pos, faces = planning_map(A)
    infl = A.InflationLayer(mm)
    infl.waveCostInflation([5, 40]); infl.vectorMap()
    n = 1000
    pts = pos[np.arange(n) % mm.V]
    fq = (np.arange(n, dtype=np.uint32) * 3) % mm.F
    bary = np.full((n, 3), 1 / 3, np.float32)
    mm.locate(pts); infl.vectorAt(fq, bary)           # both work, and whatever they leave behind is there before the probe
    before = allocated(mm.L)
    limit(10000)            # mnb_locate: the keys (8 n bytes) fit, the staged points (12 n) do not
    fails_with_cuda_error(A, lambda: mm.locate(pts))
    assert allocated(mm.L) == before
    limit(8000)             # mnb_inflation_vector_at: the faces (4 n bytes) fit, the barycentric coordinates (12 n) do not
    fails_with_cuda_error(A, lambda: infl.vectorAt(fq, bary))
    assert allocated(mm.L) == before
    limit()
    mm.close()


def failed_bvh_build(A, O):
    mm, pos, faces = planning_map(A)
    o = (pos[:50] + [0, 0, 1]).astype(np.float32)
    down = np.array([0, 0, -1], np.float32)
    before = allocated(mm.L)
    limit(2000)             # below the node arrays of the tree (2F - 1 boxes of 16 bytes)
    fails_with_cuda_error(A, lambda: mm.castRays(o, down))
    assert allocated(mm.L) == before
    limit()
    got, ref = mm.castRays(o, down), O.OracleMesh(pos, faces).cast_rays(o, down)
    assert (got["hit"] == ref["hit"]).all() and (got["face"] == ref["face"]).all() and same_bits(got["dist"], ref["dist"])
    assert int(ref["hit"].sum()) > 40
    mm.close()


def call_every_entry_point(A, mm, pos, faces):
    V = mm.V
    sf, sp = seeds_of(pos, faces, 3)
    targets = np.array([1, V // 2, V - 1], np.uint32)
    mm.computeEdgeWeights(np.zeros(V, np.float32), 1.0)
    dij, cvp, infl, obst = A.DijkstraMeshPlanner(mm), A.CVPMeshPlanner(mm), A.InflationLayer(mm), A.ObstacleLayer(mm)
    dij.dijkstra(3); dij.dijkstraBatch([3, 9]); dij.costMatrix([3, 9], targets)
    plan = cvp.waveFrontPropagation(int(sf[0]), sp[0])
    cvp.backtrack(pos[faces[sf[1]]].mean(0), int(sf[1]), max_points=500)
    mm.vectorMap(plan["pred"], plan["direction"], plan["cutting_face"])
    assert mm._check(mm.L.mnb_vector_map(mm._ctx, None, None, None, A._p(np.empty((V, 3), np.float32)))) == 0
    cvp.waveFrontPropagationBatch(sf, sp); cvp.waveFrontPropagationBatchFields(sf, sp); cvp.costMatrix(sf, sp, targets)
    mm.locate(pos[:5])
    mm.computeLayers(clearance=mm.normalClearance())
    mm.castRays(pos[:5] + np.array([0, 0, 1], np.float32), np.array([0, 0, -1], np.float32))
    obst.processPointCloud(pos[:20] + np.array([0, 0, 0.3], np.float32), want_costs=True)
    infl.waveCostInflation([5, 40], invalid=np.zeros(V, np.uint8))
    infl.onInputChanged([5, 41])
    infl.vectorMap(); infl.vectorAt(sf, np.full((3, 3), 1 / 3, np.float32))
    mm.layerChanged([2, 3], [0.5, 0.25], 1.0)
    layers = [np.full(V, 0.1, np.float32), np.full(V, 0.2, np.float32)]
    lethal = [np.zeros(V, np.uint8), np.zeros(V, np.uint8)]
    mm.maxCombinationUpdate(layers, [0.0, 0.0], lethal, [2, 3], np.zeros(V, np.float32), np.zeros(V, np.uint8))
    mm.avgCombinationUpdate(layers, [0.0, 0.0], [0.5, 0.5], lethal, [2, 3], np.zeros(V, np.float32), np.zeros(V, np.uint8))


def nothing_forgotten(A, O):
    from mesh_navigation_b200 import synth
    small_pos, small_faces = synth.grid_mesh(6, 6, terrain=True, seed=3)
    L = A._lib.load()
    start = allocated(L)
    fresh = A.MeshMap(small_pos, small_faces)
    fresh_bytes = allocated(L) - start
    fresh.close()
    assert allocated(L) == start
    mm, pos, faces = planning_map(A, 14)
    call_every_entry_point(A, mm, pos, faces)
    assert allocated(L) - start > 4 * fresh_bytes
    mm._check(L.mnb_set_mesh(mm._ctx, small_pos.shape[0], small_faces.shape[0], A._p(small_pos), A._p(small_faces), None, 0))
    # what outlives a mesh is the staging that a call sizes and the mesh does not: seed faces, seed positions, lethal vertices
    assert allocated(L) - start <= fresh_bytes + 3 * PAGE
    mm.close()
    assert allocated(L) == start


SCENARIOS = {f.__name__: f for f in (stale_seed_capacity, stale_ray_staging_capacity, stale_output_capacity,
                                     no_leak_on_error_return, failed_bvh_build, nothing_forgotten)}

if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from mesh_navigation_b200 import _lib
    _lib.LIB_PATH = EMU_LIB
    from mesh_navigation_b200 import api
    from oracle import oracle
    oracle.build()
    SCENARIOS[sys.argv[1]](api, oracle)
    print("scenario ok")
    sys.exit(0)


# ---- the tests (parent process) ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu")])
    return EMU_LIB


@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_host_memory_on_the_cpu_interpreter(emu_lib, scenario):
    env = dict(os.environ, MNB_EMU_SMS="4")
    env.pop("MNB_EMU_MALLOC_LIMIT", None)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), scenario], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and "scenario ok" in r.stdout, f"{scenario} (exit code {r.returncode}):\n{(r.stdout + r.stderr)[-3000:]}"
