"""GPU parity tests of the incremental-update entry points (SURVEY.md 3.4 / 8f3): MeshMap::layerChanged +
updateEdgeWeights, MaxCombinationLayer::onInputChanged, InflationLayer::onInputChanged -- through the C ABI, against the
oracle's restatements.  (Also replayed on the CPU interpreter of the kernels by tests/test_emu_kernels.py.)"""
import numpy as np
import pytest

from tests.util import centre_seed, disc_lethals, mesh_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _plans(api, mm, pos, faces):
    v, f, sp = centre_seed(pos, faces, (0.4, 0.6))
    c = api.CVPMeshPlanner(mm, cost_limit=2.0).waveFrontPropagation(f, sp)
    d = api.DijkstraMeshPlanner(mm, cost_limit=2.0).dijkstra(v)
    return c, d


@pytest.mark.parametrize("n,terrain,factor,frac", [(60, True, 1.5, 0.02), (90, False, 3.0, 0.2), (48, True, 0.0, 0.1)])
def test_layer_changed_matches_full_reinstall(api, oracle_mod, n, terrain, factor, frac):
    """after mnb_update_vertex_costs the device holds exactly what the oracle's layerChanged + updateEdgeWeights produce,
    and the planners (whose corner / ELL / adjacency tables were patched in place) give bit-identical fields to a map
    freshly installed with those arrays"""
    O = oracle_mod
    pos, faces = mesh_case(n, terrain)
    om = O.OracleMesh(pos, faces)
    rng = np.random.default_rng(11)
    ed = om.edge_distances()
    vc = (rng.random(om.V) * 0.8).astype(np.float32)
    w = om.edge_weights(vc, ed, factor)
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w)
    changed = rng.choice(om.V, max(1, int(frac * om.V)), replace=False).astype(np.uint32)
    new = (rng.random(changed.size) * 1.2).astype(np.float32)
    new[::17] = np.inf                                      # +inf endpoint -> +inf weight (mesh_map.cpp:598)
    layer = np.full(om.V, np.nan, np.float32); layer[changed] = new
    # oracle
    vc_ref = vc.copy(); O.layer_changed(layer, 0.0, changed, vc_ref)
    w_ref = w.copy(); om.update_edge_weights(vc_ref, ed, factor, changed, w_ref)
    # device, per-changed-vertex values; duplicates in the list are allowed
    ch_dup = np.concatenate([changed, changed[:5]]); new_dup = np.concatenate([new, new[:5]])
    mm.layerChanged(ch_dup, new_dup, factor)
    gvc, gw = mm.costs()
    assert (gvc.view(np.uint32) == vc_ref.view(np.uint32)).all()
    assert (gw.view(np.uint32) == w_ref.view(np.uint32)).all()
    if factor == 0.0:
        assert (gw.view(np.uint32) == w.view(np.uint32)).all(), "zero factor must leave the weights alone (mesh_map.cpp:568)"
    got_c, got_d = _plans(api, mm, pos, faces)
    fresh = api.MeshMap(pos, faces)
    fresh.setCosts(vc_ref, w_ref)
    ref_c, ref_d = _plans(api, fresh, pos, faces)
    for k in ("dist", "direction"):
        assert (got_c[k].view(np.uint32) == ref_c[k].view(np.uint32)).all(), k
    assert (got_c["pred"] == ref_c["pred"]).all() and (got_c["cutting_face"] == ref_c["cutting_face"]).all()
    assert (got_d["dist"].view(np.uint32) == ref_d["dist"].view(np.uint32)).all() and (got_d["pred"] == ref_d["pred"]).all()
    # and against the oracle itself
    v, f, sp = centre_seed(pos, faces, (0.4, 0.6))
    oc = om.cvp(w_ref, vc_ref, f, sp, cost_limit=2.0)
    assert (got_c["dist"].view(np.uint32) == oc["dist"].view(np.uint32)).all()
    # the V-sized-map form gives the same result
    mm2 = api.MeshMap(pos, faces); mm2.setCosts(vc, w)
    mm2.layerChanged(changed, layer, factor, by_vertex=True, default_value=0.0)
    g2, w2 = mm2.costs()
    assert (g2.view(np.uint32) == vc_ref.view(np.uint32)).all() and (w2.view(np.uint32) == w_ref.view(np.uint32)).all()
    for m in (mm, mm2, fresh):
        m.close()


def test_max_combination_update(api, oracle_mod):
    O = oracle_mod
    pos, faces = mesh_case(50, True)
    V = pos.shape[0]
    rng = np.random.default_rng(3)
    la = rng.random(V).astype(np.float32)
    lb = np.full(V, np.nan, np.float32); idx = rng.choice(V, V // 3, replace=False); lb[idx] = (rng.random(idx.size) * 2).astype(np.float32)
    lc = np.full(V, np.nan, np.float32)
    leth_a = (la > 0.9).astype(np.uint8); leth_b = (np.nan_to_num(lb) > 1.0).astype(np.uint8)
    changed = rng.choice(V, V // 4, replace=False).astype(np.uint32)
    ref_c = np.full(V, -1.0, np.float32); ref_l = np.full(V, 7, np.uint8)
    O.max_combination_update([la, lb, lc], [0.0, 0.0, 0.25], [leth_a, leth_b, None], changed, ref_c, ref_l)
    mm = api.MeshMap(pos, faces)
    got_c = np.full(V, -1.0, np.float32); got_l = np.full(V, 7, np.uint8)
    mm.maxCombinationUpdate([la, lb, lc], [0.0, 0.0, 0.25], [leth_a, leth_b, None], changed, got_c, got_l)
    assert (got_c.view(np.uint32) == ref_c.view(np.uint32)).all() and (got_l == ref_l).all()
    untouched = np.setdiff1d(np.arange(V), changed)
    assert (got_c[untouched] == -1.0).all() and (got_l[untouched] == 7).all()
    # AvgCombinationLayer (combination_layer.cpp:185-302): weighted sum in layer order; all vertices = computeLayer
    wts = [0.5, 0.3, 0.2]
    allv = np.arange(V, dtype=np.uint32)
    ref_a = np.zeros(V, np.float32); ref_al = np.zeros(V, np.uint8)
    O.avg_combination_update([la, lb, lc], [0.0, 0.1, 0.25], wts, [leth_a, leth_b, None], allv, ref_a, ref_al)
    got_a = np.zeros(V, np.float32); got_al = np.zeros(V, np.uint8)
    mm.avgCombinationUpdate([la, lb, lc], [0.0, 0.1, 0.25], wts, [leth_a, leth_b, None], allv, got_a, got_al)
    assert (got_a.view(np.uint32) == ref_a.view(np.uint32)).all() and (got_al == ref_al).all()
    assert (ref_al == (leth_a | leth_b)).all()
    mm.close()


def test_inflation_on_input_changed_chain(api, oracle_mod):
    """dynamic obstacle cycle (SURVEY 3.4): obstacles appear, move, disappear.  Every cycle: re-inflation + update set,
    final = max(static, riskiness) on the update set, layerChanged on the planner map; the planner then sees exactly the
    field a from-scratch install would give."""
    O = oracle_mod
    n = 72
    pos, faces = mesh_case(n, True)
    om = O.OracleMesh(pos, faces)
    V = om.V
    ed = om.edge_distances()
    rng = np.random.default_rng(5)
    static = (rng.random(V) * 0.3).astype(np.float32)
    factor = 2.0
    mm = api.MeshMap(pos, faces)
    vc_ref = static.copy(); w_ref = om.edge_weights(vc_ref, ed, factor)
    mm.setCosts(vc_ref, w_ref)
    infl = api.InflationLayer(mm)
    final_ref = static.copy(); final_got = static.copy()
    old_cost = None
    for cyc, (discs, seed) in enumerate([(5, 1), (5, 2), (0, 0), (9, 4)]):
        lethals = disc_lethals(pos, discs, 0.25, seed=seed) if discs else np.empty(0, np.uint32)
        ref = om.inflation(ed, lethals)
        upd_ref = O.inflation_update_set(ref["cost"], old_cost)
        got = infl.onInputChanged(lethals)
        assert (got["changed"] == upd_ref).all(), f"cycle {cyc}: update set differs"
        assert np.array_equal(np.isnan(got["cost"]), np.isnan(ref["cost"]))
        fin = ~np.isnan(ref["cost"])
        assert np.allclose(got["cost"][fin], ref["cost"][fin], rtol=1e-5, atol=0)
        old_cost = ref["cost"]
        # final combination layer on the update set, from the DEVICE's riskiness so that both sides see identical inputs
        O.max_combination_update([static, got["cost"]], [0.0, 0.0], [None, None], upd_ref, final_ref, None)
        mm.maxCombinationUpdate([static, got["cost"]], [0.0, 0.0], None, got["changed"], final_got, None)
        assert (final_got.view(np.uint32) == final_ref.view(np.uint32)).all()
        O.layer_changed(final_ref, 0.0, upd_ref, vc_ref)
        om.update_edge_weights(vc_ref, ed, factor, upd_ref, w_ref)
        mm.layerChanged(got["changed"], final_got, factor, by_vertex=True)
        gvc, gw = mm.costs()
        assert (gvc.view(np.uint32) == vc_ref.view(np.uint32)).all() and (gw.view(np.uint32) == w_ref.view(np.uint32)).all()
        v, f, sp = centre_seed(pos, faces, (0.5, 0.5))
        oc = om.cvp(w_ref, vc_ref, f, sp, cost_limit=0.9)
        gc = api.CVPMeshPlanner(mm, cost_limit=0.9).waveFrontPropagation(f, sp)
        assert (gc["dist"].view(np.uint32) == oc["dist"].view(np.uint32)).all(), f"cycle {cyc}: plan differs"
    mm.close()


@pytest.mark.parametrize("n,terrain,discs,rad,with_invalid", [(64, True, 6, 0.3, False), (90, False, 12, 0.25, True), (40, True, 2, 0.6, False)])
def test_inflation_vector_field(api, oracle_mod, n, terrain, discs, rad, with_invalid):
    """InflationLayer::vector_map_ (inflation_layer.cpp:277-308): the order-dependent accumulation of the sequential loop,
    reproduced from the final labels (ordered fold over the lethal-phase events + last accepted face)"""
    O = oracle_mod
    pos, faces = mesh_case(n, terrain)
    om = O.OracleMesh(pos, faces)
    ed = om.edge_distances()
    lethals = disc_lethals(pos, discs, rad, seed=3)
    invalid = None
    if with_invalid:
        rng = np.random.default_rng(2)
        invalid = (rng.random(om.V) < 0.03).astype(np.uint8)
        invalid[lethals[::3]] = 1                     # lethal AND invalid: fixed at the start, never expands
    ref = om.inflation(ed, lethals, invalid=invalid, inflation_radius=0.6, with_vectors=True)
    mm = api.MeshMap(pos, faces)
    infl = api.InflationLayer(mm, inflation_radius=0.6)
    got = infl.waveCostInflation(lethals, invalid)
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    vec = infl.vectorMap()
    assert np.abs(ref["vectors"]).sum() > 0
    bad = np.where((vec.view(np.uint32) != ref["vectors"].view(np.uint32)).any(1))[0]
    assert bad.size == 0, f"{bad.size} vectors differ, first {bad[:5]}: {vec[bad[:3]]} vs {ref['vectors'][bad[:3]]}"
    # vectorAt on random (face, barycentric) samples
    rng = np.random.default_rng(9)
    fq = rng.integers(0, om.F, 500).astype(np.uint32)
    b = rng.random((500, 3)).astype(np.float32); b /= b.sum(1, keepdims=True)
    gv = infl.vectorAt(fq, b)
    rv = om.inflation_vector_at(fq, b, ref["dist"], ref["vectors"], inflation_radius=0.6)
    assert np.abs(rv).sum() > 0
    assert np.allclose(gv, rv, rtol=0, atol=2e-6)
    # the labels are gone after a plan: asking again must fail loudly, the resident field stays usable
    mm.setCosts(np.zeros(om.V, np.float32), ed)
    v, f, sp = centre_seed(pos, faces, (0.5, 0.5))
    api.CVPMeshPlanner(mm).waveFrontPropagation(f, sp)
    with pytest.raises(api.MeshNavError):
        infl.vectorMap()
    assert np.allclose(infl.vectorAt(fq[:10], b[:10]), rv[:10], rtol=0, atol=2e-6)
    mm.close()


def test_backtrack_with_repulsive_field(api, oracle_mod):
    """MeshMap::meshAhead adds the layers' vectorAt (mesh_map.cpp:1097-1102): the walk bends away from the obstacles"""
    O = oracle_mod
    n = 80
    pos, faces = mesh_case(n, True)
    om = O.OracleMesh(pos, faces)
    ed = om.edge_distances()
    lethals = disc_lethals(pos, 40, 0.3, seed=12)
    ref_i = om.inflation(ed, lethals, with_vectors=True)
    vc = np.zeros(om.V, np.float32)              # the plan ignores the obstacles: the walk crosses the inflated zones
    w = om.edge_weights(vc, ed, 0.0)
    mm = api.MeshMap(pos, faces)
    infl = api.InflationLayer(mm)
    infl.waveCostInflation(lethals)
    infl.vectorMap()
    mm.setCosts(vc, w)
    planner = api.CVPMeshPlanner(mm, cost_limit=0.95)
    v, gf, gp = centre_seed(pos, faces, (0.15, 0.2))
    rv, rf, rp = centre_seed(pos, faces, (0.85, 0.8))
    plan = planner.waveFrontPropagation(gf, gp, rf)
    assert plan["outcome"] == 0
    vm = planner.computeVectorMap(plan["pred"], plan["direction"], plan["cutting_face"])
    plain = planner.backtrack(rp, rf)
    infl.setRepulsiveField(True)
    bent = planner.backtrack(rp, rf)
    infl.setRepulsiveField(False)
    rep = dict(dist=ref_i["dist"], vectors=ref_i["vectors"])
    rc0, p0, f0 = om.cvp_backtrack(vm, gp, gf, rp, rf)
    rc1, p1, f1 = om.cvp_backtrack(vm, gp, gf, rp, rf, repulsive=rep)
    assert plain["outcome"] == rc0 == 0 and bent["outcome"] == rc1
    assert plain["positions"].shape == p0.shape and np.allclose(plain["positions"], p0, atol=1e-3)
    assert bent["positions"].shape == p1.shape and np.allclose(bent["positions"], p1, atol=2e-3)
    k = min(len(p0), len(p1))
    assert np.abs(p0[:k] - p1[:k]).max() > 1e-3, "the repulsive field left the path unchanged"
    mm.close()


@pytest.mark.parametrize("n,factor", [(160, 0.0), (200, 2.0)])
def test_clean_candidate_skip_is_exact(api, oracle_mod, n, factor):
    """the batch round loop (batch_engine.cuh) carries candidates whose inputs cannot have changed over without evaluating
    them -- same potentials bit for bit as the oracle, about half the evaluations; single plans evaluate everything"""
    O = oracle_mod
    pos, faces = mesh_case(n, True)
    om = O.OracleMesh(pos, faces)
    ed = om.edge_distances()
    rng = np.random.default_rng(4)
    vc = (rng.random(om.V) * 0.7).astype(np.float32) if factor else np.zeros(om.V, np.float32)
    w = om.edge_weights(vc, ed, factor)
    v, f, sp = centre_seed(pos, faces, (0.3, 0.4))
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w)
    planner = api.CVPMeshPlanner(mm)
    base = planner.waveFrontPropagation(f, sp)
    assert base["skipped"] == 0
    sfs = np.array([f, f + 2, f + 40], np.uint32); sps = pos[faces[sfs]].mean(1).astype(np.float32)
    for cluster in (1, 2):
        mm.set_tuning(0.0, cluster, 0)
        b = planner.waveFrontPropagationBatch(sfs, sps)
        assert b["skipped"] > 0 and b["recomputes"] < 0.75 * 3 * base["recomputes"]
        for k in range(3):
            rk = om.cvp(w, vc, int(sfs[k]), sps[k])
            assert (b["dist"][k].view(np.uint32) == rk["dist"].view(np.uint32)).all(), (cluster, k)
    mm.close()


def test_layers_shared_memory_variant_is_identical(api, oracle_mod):
    """the prefetching walks of k_layers (seen-set and stack in shared memory; mode 2: 32-bit ids, mode 5: the compact
    16-bit form) against the thread-local walk (mode 0): same traversal order, so every output is bit-identical, including
    on an irregular mesh whose hub overflows into the fallback; no other mode is accepted"""
    import ctypes as C
    from tests.util import delaunay_mesh
    # third mesh: a 200 x 200 terrain with randomly permuted vertex ids -- neighbour ids differ by up to 40 000, beyond the
    # 16-bit codes of mode 5, so its per-vertex fallback runs next to the compact path
    p3, f3 = mesh_case(200, True)
    perm = np.random.default_rng(9).permutation(p3.shape[0]).astype(np.uint32)
    q3 = np.empty_like(p3); q3[perm] = p3
    for pos, faces in (mesh_case(70, True), delaunay_mesh(1500, seed=5), (q3, perm[f3])):
        mm = api.MeshMap(pos, faces)
        mm.L.mnb_debug_set_layers_smem.argtypes = [C.c_void_p, C.c_int32]
        P = api._lib.LayerParams.defaults()
        mm.L.mnb_debug_set_layers_smem(mm._ctx, 0)
        base = mm.computeLayers(P)
        P2 = api._lib.LayerParams.defaults(); P2.roughness_radius = 0.2; P2.ridge_radius = 0.45      # three separate walks
        b2 = mm.computeLayers(P2)
        for mode in (-1, 1, 3, 4, 6, 7, 8, 9, 10):
            assert mm.L.mnb_debug_set_layers_smem(mm._ctx, mode) == -1, mode      # MNB_E_ARG
        for mode in (2, 5):
            assert mm.L.mnb_debug_set_layers_smem(mm._ctx, mode) == 0
            got = mm.computeLayers(P)
            for k in list(api._lib.LAYER_NAMES) + ["combined"]:
                assert (got[k].view(np.uint32) == base[k].view(np.uint32)).all(), (mode, k)
            assert (got["lethal_mask"] == base["lethal_mask"]).all()
            g2 = mm.computeLayers(P2)
            for k in list(api._lib.LAYER_NAMES) + ["combined"]:
                assert (g2[k].view(np.uint32) == b2[k].view(np.uint32)).all(), (mode, k)
        mm.close()


def test_inflation_high_degree_vertex(api, oracle_mod):
    """a non-lethal hub with 24 incident faces, all of them usable (every ring vertex labelled): the wave must consider
    all of them, not just the first 12 of the corner list"""
    from tests.util import delaunay_mesh
    pos, faces = delaunay_mesh(3000, seed=11)
    om = oracle_mod.OracleMesh(pos, faces)
    hub = om.V - 1
    assert np.bincount(faces.reshape(-1))[hub] >= 24
    ed = om.edge_distances()
    mm = api.MeshMap(pos, faces)
    c = pos[hub, :2]
    for k, ang in enumerate(np.linspace(0.3, 6.0, 7)):
        # lethal patch just outside the hub's ring (radius 0.22), from different sides: the winning face of the hub changes
        centre = c + 0.42 * np.array([np.cos(ang), np.sin(ang)])
        le = np.where(np.linalg.norm(pos[:, :2] - centre, axis=1) < 0.17)[0].astype(np.uint32)
        assert le.size > 0 and hub not in le
        ref = om.inflation(ed, le, inflation_radius=1.2, with_vectors=True)
        infl = api.InflationLayer(mm, inflation_radius=1.2)
        got = infl.waveCostInflation(le)
        assert np.isfinite(ref["dist"][hub])
        assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all(), (k, got["dist"][hub], ref["dist"][hub])
        vec = infl.vectorMap()
        assert (vec.view(np.uint32) == ref["vectors"].view(np.uint32)).all(), k
    mm.close()


def test_update_api_edge_cases(api, oracle_mod):
    """empty / out-of-range / out-of-order uses of the incremental entry points fail loudly or are no-ops, as documented"""
    import ctypes as C
    pos, faces = mesh_case(30, True)
    om = oracle_mod.OracleMesh(pos, faces)
    V = om.V
    mm = api.MeshMap(pos, faces)
    L, ctx = mm.L, mm._ctx
    ids = np.array([1, 2], np.uint32); vals = np.array([0.5, 0.25], np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    # before the planner inputs exist
    assert L.mnb_update_vertex_costs(ctx, 2, p(ids), p(vals), 0, 0.0, 1.0) == -3                 # MNB_E_STATE
    assert L.mnb_get_costs(ctx, None, None) == -3
    assert L.mnb_inflation_vector_map(ctx, None) == -3 and L.mnb_set_repulsive_field(ctx, 1) == -3
    assert L.mnb_set_repulsive_field(ctx, 0) == 0
    ed = om.edge_distances(); vc = np.zeros(V, np.float32)
    mm.setCosts(vc, ed)
    # nothing changed / ids beyond V are ignored / duplicates are fine
    assert L.mnb_update_vertex_costs(ctx, 0, None, None, 0, 0.0, 1.0) == 0
    assert L.mnb_update_vertex_costs(ctx, 2, None, p(vals), 0, 0.0, 1.0) == -1                  # MNB_E_ARG
    wild = np.array([5, V + 7, 5, 0xffffffff], np.uint32); wv = np.array([0.3, 9.0, 0.3, 9.0], np.float32)
    mm.layerChanged(wild, wv, 2.0)
    gvc, gw = mm.costs()
    vc_ref = vc.copy(); vc_ref[5] = 0.3
    w_ref = ed.copy(); om.update_edge_weights(vc_ref, ed, 2.0, np.array([5], np.uint32), w_ref)
    assert (gvc.view(np.uint32) == vc_ref.view(np.uint32)).all() and (gw.view(np.uint32) == w_ref.view(np.uint32)).all()
    # combination: layer count limits
    lc = (C.c_void_p * 1)(p(vc)); df = np.zeros(9, np.float32); io = np.zeros(V, np.float32)
    assert L.mnb_max_combination_update(ctx, 0, lc, p(df), None, 2, p(ids), p(io), None) == -1
    assert L.mnb_max_combination_update(ctx, 9, lc, p(df), None, 2, p(ids), p(io), None) == -1
    assert L.mnb_max_combination_update(ctx, 1, lc, p(df), None, 0, None, p(io), None) == 0
    # an inflation without lethals labels nothing; its update set is whatever the previous wave had labelled
    infl = api.InflationLayer(mm)
    r0 = infl.onInputChanged(np.empty(0, np.uint32))
    assert np.isnan(r0["cost"]).all() and np.isinf(r0["dist"]).all() and r0["changed"].size == 0
    assert (infl.vectorMap() == 0).all()
    le = np.array([100, 101, 130, V + 3], np.uint32)                                             # out-of-range lethal: ignored (:412)
    r1 = infl.onInputChanged(le)
    ref = om.inflation(ed, le[:3])
    assert (r1["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    keys1 = np.where(~np.isnan(ref["cost"]))[0]
    assert (r1["changed"] == keys1).all()
    r2 = infl.onInputChanged(np.empty(0, np.uint32))
    assert np.isnan(r2["cost"]).all() and (r2["changed"] == keys1).all()                         # the vanished entries are reported
    mm.close()


def _fuzz_case(name):
    import os
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", f"fuzz_{name}.npz"))
    return (d["pos"], d["faces"], d["vc"], d["w"], d["inv"], int(d["sf"]), d["sp"], int(d["rf"]), float(d["cl"]))


def test_goal_cutoff_armed_by_a_cascade_member(api, oracle_mod):
    """found by tools/emu_fuzz.py (cost-weighted Delaunay mesh, invalid vertices, cost-limit walls): the robot-face vertex that
    arms the goal cutoff is a cascade member -- it pops late with a small potential -- so vertices beyond goal_dist had
    already popped AND expanded (cvp:754 tests the goal_dist of the moment of the pop).  A time-independent cutoff left 178
    vertices unreached and reported NO_PATH_FOUND where the reference finds the path."""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz_case("cutoff_cascade")
    om = oracle_mod.OracleMesh(pos, faces)
    ref = om.cvp(w, vc, sf, sp, rf, invalid=inv, cost_limit=cl)
    assert ref["outcome"] == 0 and ref["backsteps"] > 0
    goal_dist = ref["dist"][faces[rf]].max() + 0.3
    assert (ref["dist"][np.isfinite(ref["dist"])] > goal_dist + 1.0).any()      # labelled well beyond the cutoff: expanded before it was armed
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w, inv)
    for cluster, delta in ((-1, 0.0), (1, 0.3), (4, 0.1)):
        mm.set_tuning(delta, cluster, 0)
        got = api.CVPMeshPlanner(mm, cost_limit=cl).waveFrontPropagation(sf, sp, rf)
        assert got["outcome"] == 0
        assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all(), (cluster, delta)
        assert (got["pred"] == ref["pred"]).all() and (got["cutting_face"] == ref["cutting_face"]).all()
    mm.close()


@pytest.mark.parametrize("name", ["deep_cascade_planar", "deep_cascade_delaunay", "deep_cascade_maze"])
def test_deeply_nested_cascade(api, oracle_mod, name):
    """found by tools/emu_fuzz.py: pockets behind cost-limit / invalid walls that are flooded 'from behind' by a chain of
    back-steps, each lower than the last -- cascades nested deeper than the three levels the label word holds.  Round 1
    ordered them by creation beyond level 3 (up to 4.8 % off); the level pool (band_engine.cuh) orders them exactly."""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz_case(name)
    om = oracle_mod.OracleMesh(pos, faces)
    ref = om.cvp(w, vc, sf, sp, rf, invalid=inv, cost_limit=cl)
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w, inv)
    for cluster, delta in ((-1, 0.0), (1, 0.3), (2, 1.8)):
        mm.set_tuning(delta, cluster, 0)
        got = api.CVPMeshPlanner(mm, cost_limit=cl).waveFrontPropagation(sf, sp, rf)
        assert got["outcome"] == ref["outcome"]
        assert got["deep_labels"] > 0                                         # the case does nest deeper than the label word
        assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all(), (cluster, delta)
        assert (got["pred"] == ref["pred"]).all() and (got["cutting_face"] == ref["cutting_face"]).all()
    mm.close()


def test_inflation_backstep_deep_cascade(api, oracle_mod):
    """found by tools/emu_fuzz.py (seed 52 case 54; open in round 1): a vertex of the inflation wave takes a back-step to
    0.1142 from a face that fires at 0.1154 inside a cascade four levels deep -- the same ordering defect as above"""
    import os
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "fuzz_inflation_backstep.npz"))
    pos, faces, le, rad = d["pos"], d["faces"], d["le"], float(d["rad"])
    om = oracle_mod.OracleMesh(pos, faces)
    ref = om.inflation(om.edge_distances(), le, inflation_radius=rad, with_vectors=True)
    mm = api.MeshMap(pos, faces)
    il = api.InflationLayer(mm, inflation_radius=rad)
    got = il.waveCostInflation(le)
    vec = il.vectorMap()
    mm.close()
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    assert (vec.view(np.uint32) == ref["vectors"].view(np.uint32)).all()


def test_seed_pops_after_its_neighbour(api, oracle_mod):
    """found by tools/emu_fuzz.py (round 2, seed 202 case 13): a neighbour of the seed face lies closer to the goal point than
    the farthest seed vertex, so it pops BEFORE that seed.  Seeds are fixed before they pop (cvp:719-728): the face (seed,
    neighbour) -> c fires at the neighbour's pop, not at the later pop of the seed (which, here, does not even expand: it
    lies on a cost-limit wall).  7 547 potentials downstream were off."""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz_case("seed_after_neighbour")
    inv = inv if inv.size else None
    om = oracle_mod.OracleMesh(pos, faces)
    ref = om.cvp(w, vc, sf, sp, rf, invalid=inv, cost_limit=cl)
    sd = ref["dist"][faces[sf]]
    nb = np.unique(faces[np.isin(faces, faces[sf]).any(1)])
    assert (ref["dist"][nb] < sd.max()).sum() > (sd < sd.max()).sum()          # a non-seed neighbour below the farthest seed
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w, inv)
    for cluster, delta in ((-1, 0.0), (1, 0.3)):
        mm.set_tuning(delta, cluster, 0)
        got = api.CVPMeshPlanner(mm, cost_limit=cl).waveFrontPropagation(sf, sp, rf)
        assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all(), (cluster, delta)
        assert (got["pred"] == ref["pred"]).all() and (got["cutting_face"] == ref["cutting_face"]).all()
    mm.close()


def test_inflation_never_fixed_vertex_takes_late_updates(api, oracle_mod):
    """found by tools/emu_fuzz.py (round 2, seed 204 case 130): an invalid vertex pops without being fixed
    (inflation_layer.cpp:417-422), so a face that fires AFTER its pop still lowers it; the engine used to settle it
    with the label of its own pop time"""
    import os
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "fuzz_inflation_never_fixed.npz"))
    pos, faces, le, rad, inv = d["pos"], d["faces"], d["le"], float(d["rad"]), d["inv"]
    om = oracle_mod.OracleMesh(pos, faces)
    ref = om.inflation(om.edge_distances(), le, invalid=inv, inflation_radius=rad, with_vectors=True)
    mm = api.MeshMap(pos, faces)
    il = api.InflationLayer(mm, inflation_radius=rad)
    got = il.waveCostInflation(le, inv)
    vec = il.vectorMap()
    mm.close()
    assert (got["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all()
    assert (vec.view(np.uint32) == ref["vectors"].view(np.uint32)).all()


@pytest.mark.parametrize("name", ["deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour"])
def test_batch_engine_on_the_hard_cases(api, oracle_mod, name):
    """the lean batch round loop (batch_engine.cuh: k_cvp_batch) hands everything that is not a plain causal evaluation to the
    generic 8-lane replay; on the fixtures that exercise those paths (cascades of any depth, cost-limit walls, invalid
    vertices, seeds that pop late) every field of a batch must equal the oracle's bit for bit, for every cluster size"""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz_case(name)
    inv = inv if inv.size else None
    om = oracle_mod.OracleMesh(pos, faces)
    rng = np.random.default_rng(5)
    sfs = np.concatenate([[sf], rng.integers(0, om.F, 5)]).astype(np.uint32)
    sps = np.stack([pos[faces[f]].mean(0) for f in sfs]).astype(np.float32); sps[0] = sp
    refs = [om.cvp(w, vc, int(sfs[i]), sps[i], invalid=inv, cost_limit=cl)["dist"] for i in range(len(sfs))]
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w, inv)
    for cluster, delta in ((1, 0.3), (2, 0.1), (4, 1.8), (8, 0.3)):
        mm.set_tuning(delta, cluster, 0)
        got = api.CVPMeshPlanner(mm, cost_limit=cl).waveFrontPropagationBatch(sfs, sps)
        assert got["outcome"] == 0
        for i in range(len(sfs)):
            assert (got["dist"][i].view(np.uint32) == refs[i].view(np.uint32)).all(), (cluster, delta, i)
    mm.close()


def test_abi_argument_validation_and_trivial_dijkstra(api, oracle_mod):
    """advisor findings (round 1): caller-supplied edge lists are validated (range, duplicates) like faces; a failed
    mnb_set_mesh leaves an empty context; mnb_dijkstra with start == goal (dijkstra_mesh_planner.cpp:252-255) returns the
    cleared maps instead of uninitialised buffers"""
    import ctypes as C
    pos, faces = mesh_case(12, False)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    L, ctx = mm.L, mm._ctx
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    edges = np.ascontiguousarray(om.edges, np.uint32)
    bad = edges.copy(); bad[3, 1] = om.V + 5
    assert L.mnb_set_mesh(ctx, om.V, om.F, p(pos), p(faces), p(bad), bad.shape[0]) == -1       # MNB_E_ARG: endpoint out of range
    assert L.mnb_num_vertices(ctx) == 0                                                          # nothing half-built
    dup = edges.copy(); dup[5] = dup[4]
    assert L.mnb_set_mesh(ctx, om.V, om.F, p(pos), p(faces), p(dup), dup.shape[0]) == -1
    assert L.mnb_set_mesh(ctx, om.V, om.F, p(pos), p(faces), p(edges), edges.shape[0]) == 0
    assert L.mnb_num_vertices(ctx) == om.V
    mm.close()
    mm = api.MeshMap(pos, faces)
    mm.setCosts(np.zeros(om.V, np.float32), om.edge_distances())
    got = api.DijkstraMeshPlanner(mm).dijkstra(17, 17)
    assert got["outcome"] == 0
    exp = np.full(om.V, np.inf, np.float32); exp[17] = 0.0
    assert (got["dist"] == exp).all() and (got["pred"] == np.arange(om.V)).all()
    mm.close()
