"""GPU parity tests (run with -m gpu on an H100): every call goes through the C ABI
(libmeshnav_b200.so) and is compared with the CPU oracle on the same seeded inputs.

Bars (north_star): Dijkstra distances bit-identical and predecessors bit-exact;
CVP potentials within 1e-4 relative (we additionally report/expect bit-equality,
which the engine's event-ordered replay achieves on these meshes)."""
import numpy as np
import pytest

from tests.util import centre_seed, disc_lethals, face_of_vertex, mesh_case, rel_err

pytestmark = pytest.mark.gpu

CVP_RTOL = 1e-4   # north_star: "within 1e-4 rel (CVP float)"


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def setup(api, oracle_mod, n, terrain, seed=42, costs=None, factor=0.0, invalid=None):
    pos, faces = mesh_case(n, terrain, seed)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    assert (mm.edges() == om.edges).all()
    ed = om.edge_distances()
    vc = np.zeros(om.V, np.float32) if costs is None else costs(pos).astype(np.float32)
    w = om.edge_weights(vc, ed, factor)
    gw = mm.computeEdgeWeights(vc, factor)
    assert (gw.view(np.uint32) == w.view(np.uint32)).all(), "computeEdgeWeights differs from mesh_map.cpp:539-553"
    mm.setCosts(vc, w, invalid)
    return pos, faces, om, mm, ed, vc, w


def test_edge_distances_bit_exact(api, oracle_mod):
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 80, True)
    assert (mm.edgeDistances().view(np.uint32) == ed.view(np.uint32)).all()
    mm.close()


@pytest.mark.parametrize("n,terrain,cluster", [(100, False, 1), (100, False, 8), (64, True, 2), (200, True, 16), (150, True, 4), (120, False, -1), (300, True, -1)])
def test_dijkstra_bit_exact(api, oracle_mod, n, terrain, cluster):
    """config 1: DijkstraMeshPlanner single goal, 10k planar mesh (+ terrain variants)"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, terrain)
    mm.set_tuning(0.3, cluster, 0)
    v, f, sp = centre_seed(pos, faces, (0.25, 0.25))
    ref = om.dijkstra(w, vc, v)
    got = api.DijkstraMeshPlanner(mm).dijkstra(v)
    assert got["outcome"] == ref["outcome"] == 0
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    assert (got["pred"] == ref["pred"]).all()
    mm.close()


def test_dijkstra_goal_cutoff_costs_invalid(api, oracle_mod):
    """goal_dist cutoff (:293-300), cost_limit (:302), invalid (:328), inf edge weights, NO_PATH (:358)"""
    rng = np.random.default_rng(1)
    costs = lambda pos: np.where(rng.random(pos.shape[0]) < 0.05, 1.5, rng.random(pos.shape[0]) * 0.8)
    pos, faces = mesh_case(120, True)
    invalid = (rng.random(pos.shape[0]) < 0.01).astype(np.uint8)
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 120, True, costs=costs, factor=1.0, invalid=invalid)
    v, f, sp = centre_seed(pos, faces, (0.3, 0.3))
    invalid[v] = 0
    rv, _, _ = centre_seed(pos, faces, (0.6, 0.7))
    for robot in (-1, rv):
        ref = om.dijkstra(w, vc, v, robot_vertex=robot, invalid=invalid)
        got = api.DijkstraMeshPlanner(mm).dijkstra(v, robot)
        assert got["outcome"] == ref["outcome"]
        assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
        assert (got["pred"] == ref["pred"]).all()
    # infinite vertex costs -> +inf edge weights (mesh_map.cpp:545) and a wall -> NO_PATH_FOUND
    vc2 = vc.copy(); vc2[(pos[:, 0] > 5.0) & (pos[:, 0] < 5.4)] = np.inf
    w2 = om.edge_weights(vc2, ed, 1.0)
    mm.setCosts(vc2, w2, invalid)
    ref = om.dijkstra(w2, vc2, v, robot_vertex=rv, invalid=invalid)
    got = api.DijkstraMeshPlanner(mm).dijkstra(v, rv)
    assert ref["outcome"] == 54 and got["outcome"] == 54
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all() and (got["pred"] == ref["pred"]).all()
    mm.close()


def check_cvp(got, ref, exact_aux=True):
    r = rel_err(got["dist"], ref["dist"])
    assert r.max() <= CVP_RTOL, f"max rel err {r.max():.3e}"
    neq = int((got["dist"].view(np.uint32) != ref["dist"].view(np.uint32)).sum())
    if exact_aux and neq == 0:
        assert (got["pred"] == ref["pred"]).all()
        assert (got["cutting_face"] == ref["cutting_face"]).all()
        assert np.abs(got["direction"] - ref["direction"]).max() <= 1e-5
    return neq


@pytest.mark.parametrize("n,terrain,cluster,delta", [(100, False, -1, 0.3), (160, True, -1, 0.3), (100, False, 1, 0.3), (100, False, 8, 0.3), (100, True, 8, 0.1),
                                                     (128, True, 16, 0.6), (200, True, 2, 0.3), (90, False, 4, 1.0)])
def test_cvp_full_field(api, oracle_mod, n, terrain, cluster, delta):
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, terrain)
    mm.set_tuning(delta, cluster, 0)
    v, f, sp = centre_seed(pos, faces)
    ref = om.cvp(w, vc, f, sp)
    got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
    assert got["outcome"] == ref["outcome"] == 0
    assert check_cvp(got, ref) == 0, "potentials are expected to be bit-identical on these meshes"
    assert got["settled"] <= om.V
    mm.close()


def test_cvp_seed_near_vertex_and_border(api, oracle_mod):
    """seed point almost on a vertex (very unequal seed distances) and in a corner face of the mesh"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 90, True)
    for f in (face_of_vertex(faces, 45 * 90 + 45), 0, faces.shape[0] - 1):
        tri = pos[faces[f]]
        sp = (0.98 * tri[0] + 0.01 * tri[1] + 0.01 * tri[2]).astype(np.float32)
        ref = om.cvp(w, vc, f, sp)
        got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
        check_cvp(got, ref)
    mm.close()


def test_cvp_costs_cutoff_invalid(api, oracle_mod):
    """cost_limit (cvp:757,802), edge_cost_factor weights, invalid (:760,:785), goal cutoff (:754,:763-771), outcome codes"""
    rng = np.random.default_rng(5)
    costs = lambda pos: np.where(rng.random(pos.shape[0]) < 0.04, 1.2, rng.random(pos.shape[0]) * 0.7)
    pos, faces = mesh_case(140, True)
    invalid = (rng.random(pos.shape[0]) < 0.005).astype(np.uint8)
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 140, True, costs=costs, factor=1.0, invalid=invalid)
    v, f, sp = centre_seed(pos, faces, (0.3, 0.35))
    for x in faces[f]:
        invalid[x] = 0; vc[x] = 0.1
    w = om.edge_weights(vc, ed, 1.0)
    mm.setCosts(vc, w, invalid)
    rv, rf, _ = centre_seed(pos, faces, (0.65, 0.6))
    for robot in (-1, rf):
        ref = om.cvp(w, vc, f, sp, robot_face=robot, invalid=invalid)
        got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp, robot)
        assert got["outcome"] == ref["outcome"]
        check_cvp(got, ref)
    # unreachable robot -> NO_PATH_FOUND (cvp:912-918)
    vc2 = vc.copy(); vc2[(pos[:, 0] > 6.0) & (pos[:, 0] < 6.35)] = 3.0
    w2 = om.edge_weights(vc2, ed, 1.0)
    mm.setCosts(vc2, w2, invalid)
    ref = om.cvp(w2, vc2, f, sp, robot_face=rf, invalid=invalid)
    got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp, rf)
    assert ref["outcome"] == 54 and got["outcome"] == 54
    check_cvp(got, ref)
    mm.close()


@pytest.mark.parametrize("n,factor", [(300, 1.0), (300, 2.0), (200, 3.0)])
def test_cvp_cost_weighted_non_causal(api, oracle_mod, n, factor):
    """edge_cost_factor > 0 makes the 'edge lengths' non-geometric: large non-causal back-steps (SURVEY H1),
    |t0a| > 1 (acos NaN in the reference), nested cascades below the water line."""
    rng = np.random.default_rng(5)
    costs = lambda pos: np.where(rng.random(pos.shape[0]) < 0.04, 1.2, rng.random(pos.shape[0]) * 0.7)
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, True, costs=costs, factor=factor)
    v, f, sp = centre_seed(pos, faces, (0.3, 0.35))
    for x in faces[f]:
        vc[x] = 0.1
    w = om.edge_weights(vc, ed, factor)
    mm.setCosts(vc, w)
    ref = om.cvp(w, vc, f, sp)
    assert ref["max_backstep"] > 0.2          # the case really is strongly non-causal
    for cluster in (-1, 4):
        mm.set_tuning(0.3, cluster, 0)
        got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
        assert got["rounds"] < 2 * om.V       # converged (watchdog not hit)
        check_cvp(got, ref)
    mm.close()


def test_cvp_batch_matches_single(api, oracle_mod):
    """batched potentials (config 4 shape, small): every field equals the oracle's"""
    from mesh_navigation_b200 import synth
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 100, True)
    goals = synth.batch_goal_vertices(om.V, 12, seed=1234)
    sfs = np.array([face_of_vertex(faces, g) for g in goals], np.uint32)
    sps = np.stack([pos[faces[f]].mean(0) for f in sfs]).astype(np.float32)
    mm.set_tuning(0.3, 1, 0)
    got = api.CVPMeshPlanner(mm).waveFrontPropagationBatch(sfs, sps)
    for i in range(len(goals)):
        ref = om.cvp(w, vc, int(sfs[i]), sps[i])
        assert rel_err(got["dist"][i], ref["dist"]).max() <= CVP_RTOL
    mm.close()


def test_large_mesh_properties(api, oracle_mod):
    """1M-vertex terrain (config 2): parity vs the oracle + size-independent properties."""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 1000, True)
    v, f, sp = centre_seed(pos, faces)
    got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
    ref = om.cvp(w, vc, f, sp)
    assert rel_err(got["dist"], ref["dist"]).max() <= CVP_RTOL
    d = got["dist"]
    assert np.isfinite(d).all() and got["settled"] >= om.V - 3
    eu = np.linalg.norm(pos - sp, axis=1)
    assert (d >= eu - 1e-4).all()                                    # a geodesic is never shorter than the chord
    p = got["pred"]; nz = p != np.arange(om.V)
    assert nz.sum() == om.V - 3                                      # everything but the 3 seeds has a predecessor
    gd = api.DijkstraMeshPlanner(mm).dijkstra(v)
    rd = om.dijkstra(w, vc, v)
    assert (gd["dist"].view(np.uint32) == rd["dist"].view(np.uint32)).all() and (gd["pred"] == rd["pred"]).all()
    assert (gd["dist"][gd["pred"][nz]] <= gd["dist"][nz]).all()
    # triangle inequality along every edge: |d(a) - d(b)| <= w(a,b)
    a, b = om.edges[:, 0], om.edges[:, 1]
    assert (np.abs(gd["dist"][a] - gd["dist"][b]) <= w + 2e-5).all()      # one float ulp at d ~ 100 m is 7.6e-6
    mm.close()


INFL_DIST_RTOL = 1e-4    # proposed bar (BASELINE.md config 3): inflation dist <= 1e-4 rel, costs <= 1e-5 rel


def check_inflation(got, ref, radius):
    fr, fg = np.isfinite(ref["dist"]), np.isfinite(got["dist"])
    assert (fr == fg).all(), f"labelled sets differ: only ref {(fr & ~fg).sum()}, only gpu {(fg & ~fr).sum()}"
    r = rel_err(got["dist"], ref["dist"])
    assert r.max() <= INFL_DIST_RTOL, f"max rel err {r.max():.3e}"
    assert (np.isnan(got["cost"]) == np.isnan(ref["cost"])).all()
    ok = ~np.isnan(ref["cost"])
    assert np.allclose(got["cost"][ok], ref["cost"][ok], rtol=1e-5, atol=1e-7)
    inside = fr & (ref["dist"] <= radius)
    return int((got["dist"][inside].view(np.uint32) != ref["dist"][inside].view(np.uint32)).sum())


@pytest.mark.parametrize("n,terrain,discs,rad", [(100, False, 8, 0.3), (160, True, 40, 0.3), (120, True, 10, 0.15)])
def test_inflation_wave(api, oracle_mod, n, terrain, discs, rad):
    """InflationLayer::waveCostInflation: synthetic obstacle discs (SURVEY 8d config 3), default config"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, terrain)
    assert int(np.diff(np.bincount(faces.reshape(-1))).max()) < 12
    le = disc_lethals(pos, discs, rad)
    assert le.size > 10
    ref = om.inflation(ed, le)
    got = api.InflationLayer(mm).waveCostInflation(le)
    assert check_inflation(got, ref, 0.4) == 0, "distances inside the inflation radius are expected bit-identical"
    mm.close()


def test_inflation_params_invalid_and_edge_cases(api, oracle_mod):
    """reference test config (0.5 / 1.5 / 0.9, inflation_layer_test.cpp:41-45), invalid vertices (:417),
    isolated lethal vertices (no face with two fixed vertices -> no propagation), empty lethal set"""
    rng = np.random.default_rng(11)
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 150, True)
    le = np.concatenate([disc_lethals(pos, 12, 0.35, seed=3), np.array([5, 5, 777, 12000], np.uint32)])
    invalid = (rng.random(om.V) < 0.01).astype(np.uint8)
    kw = dict(inscribed_radius=0.5, inflation_radius=1.5, lethal_value=1.0, inscribed_value=0.9, cost_scaling_factor=1.0)
    for inv in (None, invalid):
        ref = om.inflation(ed, le, invalid=inv, **kw)
        got = api.InflationLayer(mm, **kw).waveCostInflation(le, inv)
        check_inflation(got, ref, 1.5)
    ref = om.inflation(ed, np.array([4000], np.uint32))
    got = api.InflationLayer(mm).waveCostInflation(np.array([4000], np.uint32))
    assert np.isfinite(got["dist"]).sum() == np.isfinite(ref["dist"]).sum() == 1
    got = api.InflationLayer(mm).waveCostInflation(np.zeros(0, np.uint32))
    assert not np.isfinite(got["dist"]).any() and np.isnan(got["cost"]).all()
    mm.close()


LAYER_RTOL = 1e-5    # proposed bar (BASELINE.md config 3): layer costs <= 1e-5 rel


def test_geometric_layers_fused(api, oracle_mod):
    """six geometric layers + Max combination + lethal masks (a10/a11); definitions: oracle orc_layers"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 220, True)
    ref = om.layers()
    assert np.allclose(mm.vertexNormals(), ref["vertex_normals"], rtol=0, atol=1e-6)
    got = mm.computeLayers()
    for name in ("height_diff", "ridge", "clearance", "border"):      # no transcendental: bit-identical
        assert (got[name].view(np.uint32) == ref[name].view(np.uint32)).all(), name
    # acos is evaluated in double and rounded once on both sides (kernels_layers.cuh acos_f / oracle acosF): the values agree to
    # the last bit except where the two double-precision acos implementations differ in their last bit AND that straddles a
    # float rounding boundary (~1e-8 of the calls); the roughness sum may then differ by one ulp
    for name in ("roughness", "steepness", "combined"):
        assert np.allclose(got[name], ref[name], rtol=2e-7, atol=0), name
        assert (got[name].view(np.uint32) != ref[name].view(np.uint32)).mean() < 1e-4, name
    assert (got["lethal_mask"] == ref["lethal_mask"]).all()             # lethal sets identical (BASELINE.md config 3)
    assert (ref["lethal_mask"] != 0).sum() > 100
    # non-default radii (three separate walks) and a clearance input
    P = oracle_mod.LayerParams.defaults(); P.height_diff_radius = 0.25; P.ridge_radius = 0.4; P.roughness_radius = 0.2
    from mesh_navigation_b200 import _lib
    G = _lib.LayerParams.defaults(); G.height_diff_radius = 0.25; G.ridge_radius = 0.4; G.roughness_radius = 0.2
    rng = np.random.default_rng(2)
    cl = (0.3 + rng.random(om.V) * 0.8).astype(np.float32); cl[::7] = np.inf
    ref = om.layers(P, cl); got = mm.computeLayers(G, cl)
    for name in ("height_diff", "ridge", "border"):
        assert (got[name].view(np.uint32) == ref[name].view(np.uint32)).all(), name
    assert np.allclose(got["clearance"], ref["clearance"], rtol=1e-6, atol=1e-7)
    assert ((got["lethal_mask"] & 16) == (ref["lethal_mask"] & 16)).all()
    mm.close()


def test_config3_layer_stack_chain(api, oracle_mod):
    """config 3 chain: layers -> Max combination -> lethals (+ obstacle discs) -> waveCostInflation ->
    vertex_costs -> computeEdgeWeights (factor 1.0) -> CVP plan; every stage checked against the oracle"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 250, True)
    ref_l = om.layers(); got_l = mm.computeLayers()
    lethal_ref = np.union1d(np.where(ref_l["lethal_mask"] != 0)[0], disc_lethals(pos, 15, 0.3)).astype(np.uint32)
    lethal_got = np.union1d(np.where(got_l["lethal_mask"] != 0)[0], disc_lethals(pos, 15, 0.3)).astype(np.uint32)
    assert np.array_equal(lethal_ref, lethal_got)                       # lethal sets identical
    ref_i = om.inflation(ed, lethal_ref); got_i = api.InflationLayer(mm).waveCostInflation(lethal_ref)
    check_inflation(got_i, ref_i, 0.4)
    vcost = np.where(np.isnan(ref_i["cost"]), 0.0, ref_i["cost"]).astype(np.float32)   # InflationLayer default value 0
    w1 = om.edge_weights(vcost, ed, 1.0)
    gw = mm.computeEdgeWeights(vcost, 1.0)
    assert (gw.view(np.uint32) == w1.view(np.uint32)).all()
    v, f, sp = centre_seed(pos, faces, (0.5, 0.5))
    free = np.where(vcost < 0.5)[0]
    v = int(free[np.argmin(np.linalg.norm(pos[free] - pos[v], axis=1))]); f = face_of_vertex(faces, v)
    while not (vcost[faces[f]] < 1.0).all():
        f += 1
    sp = pos[faces[f]].mean(0).astype(np.float32)
    ref = om.cvp(w1, vcost, f, sp)
    got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
    check_cvp(got, ref)
    assert np.isfinite(ref["dist"]).sum() > 0.5 * om.V
    mm.close()


def test_irregular_mesh_all_paths(api, oracle_mod):
    """Delaunay mesh with vertex degrees 3..24: exercises the ELL overflow (> 8 faces) and the rescanning replay
    (> 12 faces) paths, a mesh boundary everywhere and strongly varying triangle shapes."""
    from tests.util import delaunay_mesh
    pos, faces = delaunay_mesh(6000)
    om = oracle_mod.OracleMesh(pos, faces)
    deg = np.bincount(faces.reshape(-1))
    assert deg.max() >= 24 and (deg > 8).sum() > 20
    mm = api.MeshMap(pos, faces)
    assert (mm.edges() == om.edges).all()
    ed = om.edge_distances()
    assert (mm.edgeDistances().view(np.uint32) == ed.view(np.uint32)).all()
    rng = np.random.default_rng(9)
    vc = (rng.random(om.V) * 0.6).astype(np.float32)
    for factor in (0.0, 1.0):
        w = om.edge_weights(vc, ed, factor)
        assert (mm.computeEdgeWeights(vc, factor).view(np.uint32) == w.view(np.uint32)).all()
        hub = om.V - 1
        seeds = [hub, int(np.argmin(np.linalg.norm(pos[:, :2] - [1.0, 1.0], axis=1)))]
        for sv in seeds:
            ref = om.dijkstra(w, vc, sv); got = api.DijkstraMeshPlanner(mm).dijkstra(sv)
            assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all() and (got["pred"] == ref["pred"]).all()
            f = face_of_vertex(faces, sv); sp = pos[faces[f]].mean(0).astype(np.float32)
            ref = om.cvp(w, vc, f, sp)
            for cluster in (-1, 2):
                mm.set_tuning(0.3, cluster, 0)
                got = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
                check_cvp(got, ref)
    # inflation + layers on the irregular mesh
    le = np.where(np.linalg.norm(pos[:, :2] - [3.0, 3.0], axis=1) < 0.5)[0].astype(np.uint32)
    ref = om.inflation(ed, le); got = api.InflationLayer(mm).waveCostInflation(le)
    check_inflation(got, ref, 0.4)
    le2 = np.where(np.linalg.norm(pos[:, :2] - pos[om.V - 1, :2], axis=1) < 0.25)[0].astype(np.uint32)   # around the hub
    ref = om.inflation(ed, le2); got = api.InflationLayer(mm).waveCostInflation(le2)
    check_inflation(got, ref, 0.4)
    refl = om.layers(); gotl = mm.computeLayers()
    for name in ("height_diff", "ridge", "border"):
        assert (gotl[name].view(np.uint32) == refl[name].view(np.uint32)).all(), name
    assert np.allclose(gotl["roughness"], refl["roughness"], rtol=LAYER_RTOL, atol=1e-6)
    mm.close()


def test_disconnected_and_tiny_meshes(api, oracle_mod):
    """two disconnected components (unreachable part stays +inf / pred self), and the single-triangle mesh of the
    reference's own test (inflation_layer_test.cpp:7-23)"""
    pos1, faces1 = mesh_case(20, False)
    pos2 = pos1 + np.array([10.0, 0, 0], np.float32)
    pos = np.concatenate([pos1, pos2]); faces = np.concatenate([faces1, faces1 + len(pos1)]).astype(np.uint32)
    om = oracle_mod.OracleMesh(pos, faces); mm = api.MeshMap(pos, faces)
    ed = om.edge_distances(); vc = np.zeros(om.V, np.float32); mm.setCosts(vc, ed)
    ref = om.cvp(ed, vc, 10, pos[faces[10]].mean(0)); got = api.CVPMeshPlanner(mm).waveFrontPropagation(10, pos[faces[10]].mean(0))
    check_cvp(got, ref)
    assert np.isinf(got["dist"][len(pos1):]).all() and (got["pred"][len(pos1):] == np.arange(len(pos1), om.V)).all()
    refd = om.dijkstra(ed, vc, 5, robot_vertex=len(pos1) + 3); gotd = api.DijkstraMeshPlanner(mm).dijkstra(5, len(pos1) + 3)
    assert refd["outcome"] == gotd["outcome"] == 54
    assert (gotd["dist"].view(np.uint32) == refd["dist"].view(np.uint32)).all()
    mm.close()
    tri_pos = np.array([[0, 0, 0], [0.5, 0, 0], [0, 0.5, 0]], np.float32); tri = np.array([[0, 1, 2]], np.uint32)
    om = oracle_mod.OracleMesh(tri_pos, tri); mm = api.MeshMap(tri_pos, tri)
    ed = om.edge_distances(); mm.setCosts(np.zeros(3, np.float32), ed)
    got = api.DijkstraMeshPlanner(mm).dijkstra(0)
    assert got["dist"].tolist() == [0.0, 0.5, 0.5] and got["pred"].tolist() == [0, 0, 0]
    got = api.CVPMeshPlanner(mm).waveFrontPropagation(0, np.array([0.1, 0.1, 0.0], np.float32))
    ref = om.cvp(ed, np.zeros(3, np.float32), 0, np.array([0.1, 0.1, 0.0], np.float32))
    assert (got["dist"] == ref["dist"]).all()
    # the reference's own triangle (inflation_layer_test.cpp:7-23): its known answer (d = 0, 0.5 -> 0.5) pins the ORACLE's
    # waveFrontUpdate (tests/test_oracle_golden.py); a wave needs two fixed vertices, so here both corners are lethal and the
    # kernel must reproduce the oracle's wave bit for bit
    got = api.InflationLayer(mm, 0.5, 1.5, 1.0, 0.9, 1.0).waveCostInflation(np.array([0, 1], np.uint32))
    ref = om.inflation(ed, np.array([0, 1], np.uint32), inscribed_radius=0.5, inflation_radius=1.5, lethal_value=1.0, inscribed_value=0.9,
                       cost_scaling_factor=1.0)
    assert got["dist"][:2].tolist() == [0.0, 0.0] and 0.5 <= got["dist"][2] < 0.7
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    assert (got["cost"].view(np.uint32) == ref["cost"].view(np.uint32)).all()
    mm.close()


def test_cancel_returns_canceled(api, oracle_mod):
    """mnb_cancel from another thread while a plan runs -> MBF CANCELED (51) (cvp_mesh_planner.cpp:142-146, 888-892)"""
    import threading, time
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 700, True)
    mm.set_tuning(0.02, 1, 0)          # tiny band + one CTA: a deliberately slow plan (tens of ms)
    v, f, sp = centre_seed(pos, faces)
    t0 = time.perf_counter(); full = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp); t_full = time.perf_counter() - t0
    assert full["outcome"] == 0 and t_full > 0.02, "the uncancelled plan must take long enough for the cancel to land inside it"
    outcomes = []
    def run():
        t1 = time.perf_counter(); o = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)["outcome"]; outcomes.append((o, time.perf_counter() - t1))
    t = threading.Thread(target=run)
    t.start(); time.sleep(0.25 * t_full); mm.cancel(); t.join()
    assert outcomes[0][0] == 51, outcomes                    # CANCELED: the request took effect ...
    assert outcomes[0][1] < 0.85 * t_full, (outcomes, t_full)  # ... and cut the plan short
    mm.set_tuning(0.3, -1, 0)
    assert api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)["outcome"] == 0     # the flag is reset per plan (cvp:679)
    mm.close()


def test_vector_maps(api, oracle_mod):
    """a2 DijkstraMeshPlanner::computeVectorMap (:189-209) and a6 CVPMeshPlanner::computeVectorMap (:204-239)"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 150, True)
    v, f, sp = centre_seed(pos, faces, (0.4, 0.6))
    gd = api.DijkstraMeshPlanner(mm).dijkstra(v)
    ref = om.dijkstra_vector_map(gd["pred"]); got = api.DijkstraMeshPlanner(mm).computeVectorMap(gd["pred"])
    assert (np.isnan(ref) == np.isnan(got)).all() and np.isnan(got[v]).all()
    ok = ~np.isnan(ref)
    assert (got[ok].view(np.uint32) == ref[ok].view(np.uint32)).all()                 # no transcendental: bit-identical
    gc = api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
    vn = om.layers()["vertex_normals"]
    ref = om.cvp_vector_map(vn, gc["pred"], gc["direction"], gc["cutting_face"])
    got = api.CVPMeshPlanner(mm).computeVectorMap(gc["pred"], gc["direction"], gc["cutting_face"])
    assert (np.isnan(ref) == np.isnan(got)).all()
    ok = ~np.isnan(ref)
    assert np.abs(got[ok] - ref[ok]).max() <= 2e-6                                     # sin/cos: CUDA vs glibc, last-bit
    assert np.allclose(np.linalg.norm(got.reshape(-1, 3)[~np.isnan(got).any(1)], axis=1), 1.0, atol=1e-5)
    # the field points down the potential: following it one edge towards the predecessor lowers the potential
    nz = gc["pred"] != np.arange(om.V)
    assert (gc["dist"][gc["pred"][nz]] < gc["dist"][nz] + 1e-6).mean() > 0.99
    mm.close()


def _backtrack_case(api, oracle_mod, n, weighted, seed_uv, robot_uv, terrain=True):
    costs = (lambda p: 0.45 + 0.45 * np.sin(3.0 * p[:, 0]) * np.cos(2.0 * p[:, 1])) if weighted else None
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, True, costs=costs, factor=1.0 if weighted else 0.0)
    sv, sf, sp = centre_seed(pos, faces, seed_uv)
    rv, rf, rp = centre_seed(pos, faces, robot_uv)
    pl = api.CVPMeshPlanner(mm)
    g = pl.waveFrontPropagation(sf, sp, rf)
    assert g["outcome"] == 0
    vm = pl.computeVectorMap(g["pred"], g["direction"], g["cutting_face"])
    bt = pl.backtrack(rp, rf)
    # oracle walk on the GPU's vector map: same float arithmetic, no transcendental -> bit-identical
    rc, opos, oface = om.cvp_backtrack(vm, sp, sf, rp, rf, 0.4)
    return pos, faces, om, mm, pl, g, vm, bt, (rc, opos, oface), (sf, sp, rf, rp, vc, w)


@pytest.mark.parametrize("weighted", [False, True])
def test_backtrack_parity(api, oracle_mod, weighted):
    """f1: cvp:920-951 back-tracking over MeshMap::meshAhead; GPU walk == oracle walk on the same field"""
    pos, faces, om, mm, pl, g, vm, bt, (rc, opos, oface), (sf, sp, rf, rp, vc, w) = _backtrack_case(
        api, oracle_mod, 200, weighted, (0.2, 0.25), (0.8, 0.7))
    assert rc == 0 and bt["outcome"] == 0
    assert len(bt["positions"]) == len(opos) and len(opos) > 10
    assert (bt["positions"].view(np.uint32) == opos.view(np.uint32)).all()
    assert (bt["faces"] == oface).all()
    p = bt["positions"]
    assert (p[0] == rp).all() and (p[-1] == sp).all() and bt["faces"][0] == rf and bt["faces"][-1] == sf
    seg = np.linalg.norm(np.diff(p, axis=0), axis=1)
    assert seg[:-1].max() <= 0.4 * 1.5 + 1e-3          # step_width (+ the projection onto a neighbour face)
    # the walk descends the potential: path length ~ potential at the robot (geodesic), never shorter than the chord
    length = seg.sum()
    chord = np.linalg.norm(rp - sp)
    pot_robot = g["dist"][faces[rf]].mean()
    assert chord * 0.999 <= length
    if not weighted:
        assert length <= pot_robot * 1.10 + 0.8
    # end-to-end with the oracle's own wavefront + vector map (sin/cos last-bit differences only)
    o = om.cvp(w, vc, sf, sp, rf)
    ovm = om.cvp_vector_map(om.layers()["vertex_normals"], o["pred"], o["direction"], o["cutting_face"])
    rc2, opos2, _ = om.cvp_backtrack(ovm, sp, sf, rp, rf, 0.4)
    assert rc2 == 0 and len(opos2) == len(p)
    assert np.abs(opos2 - p).max() <= 1e-3
    mm.close()


def test_make_plan_path_only(api, oracle_mod):
    """makePlan keeps the four V-sized maps on the device; the path alone crosses PCIe"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 160, False)
    gv, gf, gp = centre_seed(pos, faces, (0.75, 0.3))
    sv, sf, sp = centre_seed(pos, faces, (0.15, 0.8))
    pl = api.CVPMeshPlanner(mm)
    r = pl.makePlan(sp, sf, gp, gf)
    assert r["outcome"] == 0 and (r["positions"][0] == sp).all() and (r["positions"][-1] == gp).all()
    g = pl.waveFrontPropagation(gf, gp, sf)
    vm = pl.computeVectorMap(g["pred"], g["direction"], g["cutting_face"])
    rc, opos, oface = om.cvp_backtrack(vm, gp, gf, sp, sf, 0.4)
    assert rc == 0 and (opos.view(np.uint32) == r["positions"].view(np.uint32)).all()
    assert abs(r["cost"] - np.linalg.norm(np.diff(opos, axis=0), axis=1).sum()) < 1e-3
    mm.close()


def test_backtrack_needs_plan(api, oracle_mod):
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, 40, False)
    with pytest.raises(RuntimeError):
        api.CVPMeshPlanner(mm).backtrack(pos[0], 0)
    mm.close()


@pytest.mark.parametrize("n,nq", [(120, 1), (200, 77), (64, 300)])
def test_locate_parity(api, oracle_mod, n, nq):
    """f2: getNearestVertexHandle (mesh_map.cpp:1161-1174) + searchContainingFace (:1120-1159), batched on the GPU"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, True)
    rng = np.random.default_rng(5)
    fsel = rng.integers(0, faces.shape[0], nq)
    b = rng.dirichlet((1, 1, 1), nq).astype(np.float32)
    pts = (pos[faces[fsel]] * b[:, :, None]).sum(1).astype(np.float32)
    pts[:, 2] += rng.normal(0, 0.05, nq).astype(np.float32)            # off the surface
    pts[::7] += np.float32(50.0)                                        # far outside: nearest vertex yes, face no
    pts[::5] = pos[rng.integers(0, pos.shape[0], len(pts[::5]))]        # exactly on vertices
    ov, of, ob = om.locate(pts)
    gv, gf, gb = mm.locate(pts)
    assert (gv == ov).all() and (gf == of).all()
    assert (gb.view(np.uint32) == ob.view(np.uint32)).all()
    assert (of[::7][np.arange(len(of[::7])) % 5 != 0] == -1).all() or nq < 8
    inside = of >= 0
    assert inside.mean() > 0.5 or nq == 1
    # the reported face really contains the projected point
    assert (gb[inside] >= -0.0100001).all() and (gb[inside] <= 1.0100001).all()
    assert mm.getNearestVertexHandle(pts[0]) == ov[0] and mm.getContainingFace(pts[0]) == of[0]
    mm.close()


@pytest.mark.parametrize("n", [24, 48, 90])
def test_goal_cutoff_small_mesh_wide_band(api, oracle_mod, n):
    """goal cutoff (cvp:754,763-771 / dijkstra:293-300) when the band is wider than the whole mesh: everything settles
    before the cutoff is known and the vertices beyond it have to be put back and recomputed"""
    pos, faces, om, mm, ed, vc, w = setup(api, oracle_mod, n, True)
    sv, sf, sp = centre_seed(pos, faces, (0.3, 0.3))
    rv, rf, rp = centre_seed(pos, faces, (0.55, 0.6))
    ref = om.dijkstra(w, vc, sv, rv)
    got = api.DijkstraMeshPlanner(mm).dijkstra(sv, rv)
    assert got["outcome"] == ref["outcome"] == 0
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    assert (got["pred"] == ref["pred"]).all()
    assert np.isinf(ref["dist"]).any() or n < 60          # the cutoff really cut something off
    ref = om.cvp(w, vc, sf, sp, rf)
    got = api.CVPMeshPlanner(mm).waveFrontPropagation(sf, sp, rf)
    assert got["outcome"] == ref["outcome"] == 0
    assert rel_err(got["dist"], ref["dist"]).max() <= 1e-4
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    assert (got["pred"] == ref["pred"]).all()
    mm.close()
