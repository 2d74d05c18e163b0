"""Inflation repair (mnb_inflation_repair / InflationLayer.repairInflation): every step of a chain of lethal sets runs the
repair on one context and a full mnb_inflation_update on a second context over the same map, and compares bit for bit
(as uint32): distances and riskiness, the changed set against the bitwise diff of consecutive full results, the repulsive
field, and the update set a later full call on the repair context reports.  On the small meshes the full result is also
checked against the oracle.  The GPU tests run with -m gpu on an H100; the interpreter test replays them on the CPU
interpreter of the kernels (tests/emu), and the oracle test checks the premise of the repair (DESIGN §4) on the CPU."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from mesh_navigation_b200 import synth
from tests.util import centre_seed, delaunay_mesh, disc_lethals, mesh_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def _changed(new, old):
    """vertices whose riskiness entry differs: presence or value bits, NaN = no entry, NaN equal to NaN"""
    if old is None:
        return np.where(~np.isnan(new))[0].astype(np.uint32)
    diff = (new.view(np.uint32) != old.view(np.uint32)) & ~(np.isnan(new) & np.isnan(old))
    return np.where(diff)[0].astype(np.uint32)


def _mesh(kind):
    if kind == "terrain":
        return mesh_case(36, True)
    if kind == "planar":
        return mesh_case(36, False)
    if kind == "exact_ties":                         # unjittered planar grid: many equal candidates
        return synth.grid_mesh(34, 34, jitter=0.0, terrain=False)
    if kind in ("delaunay", "invalid"):              # the Delaunay mesh has a degree-24 hub vertex
        return delaunay_mesh(1100, seed=5, extent=3.6)
    raise ValueError(kind)


def _disc(pos, frac, r):
    """vertices within r (xy) of the point at fractions `frac` of the map's extent"""
    lo, hi = pos[:, :2].min(0), pos[:, :2].max(0)
    c = lo + (hi - lo) * np.asarray(frac, np.float64)
    return np.where(((pos[:, :2] - c) ** 2).sum(1) <= r * r)[0].astype(np.uint32)


class Pair:
    """one map on two contexts: `rep` runs repairs, `full` runs mnb_inflation_update on the same sequence.  With alt, two
    more contexts take turns: on every step one of them, whose last call was a repair, runs the full update (its update
    set must be the full context's), and the other one runs the repair."""

    def __init__(self, api, oracle_mod, pos, faces, radius=0.4, oracle=True, field=True, alt=False):
        self.api, self.pos, self.faces, self.radius, self.field = api, pos, faces, radius, field
        self.rmap, self.fmap = api.MeshMap(pos, faces), api.MeshMap(pos, faces)
        self.rep = api.InflationLayer(self.rmap, inflation_radius=radius)
        self.full = api.InflationLayer(self.fmap, inflation_radius=radius)
        self.amaps = [api.MeshMap(pos, faces) for _ in range(2)] if alt else []
        self.alt = [api.InflationLayer(m, inflation_radius=radius) for m in self.amaps]
        self.k = 0
        self.O = oracle_mod
        self.om = oracle_mod.OracleMesh(pos, faces) if oracle else None
        self.ed = self.om.edge_distances() if oracle else None
        self.V = pos.shape[0]
        self.prev = None                 # riskiness of the previous step
        self.field_valid = False         # the repair context's repulsive field is valid

    def step(self, lethals, invalid=None, repair=True):
        le = np.asarray(lethals, np.uint32)
        got = self.rep.repairInflation(le, invalid) if repair else self.rep.onInputChanged(le, invalid)
        ref = self.full.onInputChanged(le, invalid)
        assert _same(got["dist"], ref["dist"]), "dist"
        assert _same(got["cost"], ref["cost"]), "cost"
        if self.alt:
            x, y = self.alt[self.k % 2], self.alt[1 - self.k % 2]
            gx = x.onInputChanged(le, invalid)
            if self.k > 0:                           # x repaired the previous step
                assert np.array_equal(gx["changed"], ref["changed"]), "update set of a full call after a repair"
            gy = y.repairInflation(le, invalid)
            assert _same(gy["dist"], ref["dist"]) and _same(gy["cost"], ref["cost"]), "repair after a full call"
            assert np.array_equal(gy["changed"], _changed(ref["cost"], self.prev)), "changed set after a full call"
        self.k += 1
        self.ref = ref
        if repair:
            assert np.array_equal(got["changed"], _changed(ref["cost"], self.prev)), "changed set"
        else:                                        # d_prev_risk was patched: the same update set as the full chain
            assert np.array_equal(got["changed"], ref["changed"]), "update set after repairs"
        if self.field:
            ref_vec = self.full.vectorMap()
            if repair and self.field_valid:
                assert _same(self.rep.vectorMap(), ref_vec), "repulsive field"
            elif not self.field_valid or not repair:
                self.rep.vectorMap()                 # labels of a whole-map wave: the field becomes valid
                self.field_valid = True
        if self.om is not None:
            o = self.om.inflation(self.ed, le[le < self.V], invalid=invalid, inflation_radius=self.radius)
            assert np.array_equal(np.isnan(got["cost"]), np.isnan(o["cost"]))
            fin = ~np.isnan(o["cost"])
            assert np.allclose(got["cost"][fin], o["cost"][fin], rtol=1e-5, atol=0)
            assert np.array_equal(np.isfinite(got["dist"]), np.isfinite(o["dist"]))
        self.prev = ref["cost"]
        return got

    def close(self):
        for m in [self.rmap, self.fmap] + self.amaps:
            m.close()


def _invalid_mask(kind, V):
    if kind != "invalid":
        return None
    rng = np.random.default_rng(11)
    return (rng.random(V) < 0.04).astype(np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [0.4, 1.0])
@pytest.mark.parametrize("kind", ["terrain", "planar", "exact_ties", "delaunay", "invalid"])
def test_repair_chain(api, oracle_mod, kind, radius):
    """discs appear, move, touch the static lethals (a disc and the left border), merge and split, disappear; the same
    set twice; duplicates and ids >= V; no lethals; every vertex lethal"""
    pos, faces = _mesh(kind)
    V = pos.shape[0]
    inv = _invalid_mask(kind, V)
    p = Pair(api, oracle_mod, pos, faces, radius, alt=True)
    border = np.where(pos[:, 0] <= pos[:, 0].min() + 0.02)[0].astype(np.uint32)
    static = np.union1d(_disc(pos, (0.3, 0.3), 0.3), border).astype(np.uint32)
    u = lambda *sets: np.unique(np.concatenate([static, *sets])).astype(np.uint32)
    steps = [
        ("static", static),                                      # no previous result: whole-map wave
        ("appears", u(_disc(pos, (0.75, 0.7), 0.2))),
        ("moves", u(_disc(pos, (0.75, 0.76), 0.2))),
        ("touches static", u(_disc(pos, (0.3, 0.45), 0.15))),
        ("disappears", static),
        ("two apart", u(_disc(pos, (0.6, 0.2), 0.12), _disc(pos, (0.85, 0.2), 0.12))),
        ("merged", u(_disc(pos, (0.68, 0.2), 0.12), _disc(pos, (0.77, 0.2), 0.12))),
        ("split", u(_disc(pos, (0.6, 0.2), 0.12), _disc(pos, (0.85, 0.2), 0.12))),
    ]
    for name, le in steps:
        r = p.step(le, inv)
        assert r["changed"].size > 0, name
    # the same lethal set again: nothing changes and no wave runs
    r = p.step(steps[-1][1][::-1].copy(), inv)
    assert r["changed"].size == 0 and r["settled"] == 0 and r["rounds"] == 0
    # duplicates and ids >= V are ignored
    le = steps[1][1]
    p.step(np.concatenate([le, le[:7], [V, V + 5, 0xFFFFFFFF]]).astype(np.uint32), inv)
    p.step(np.empty(0, np.uint32), inv)                          # every lethal removed
    p.step(np.arange(V, dtype=np.uint32), inv)                   # every vertex lethal
    p.step(static, inv)
    p.close()


@pytest.mark.gpu
def test_repair_second_pass(api, oracle_mod):
    """a disc whose lethals are outside a static cluster's footprint but whose new footprint reaches it: the merge
    check adds the cluster and the wave runs again"""
    pos, faces = mesh_case(40, True)
    p = Pair(api, oracle_mod, pos, faces, 0.4, field=False)
    lo, hi = pos[:, :2].min(0), pos[:, :2].max(0)
    frac = lambda xy: (np.asarray(xy) - lo) / (hi - lo)
    a = _disc(pos, frac((1.0, 2.0)), 0.35)                      # larger than the disc: its cluster is the smaller share
    p.step(a)
    p.step(np.union1d(a, _disc(pos, frac((3.0, 2.0)), 0.2)))      # far away: one pass (and the first cluster ids)
    one = p.step(np.union1d(a, _disc(pos, frac((3.0, 2.2)), 0.2)))
    # one pass: the wave runs from the disc alone and settles less than the full wave from every lethal
    assert 0 < one["settled"] < p.ref["settled"]
    # lethal gap 0.78 m: more than the footprint of either side plus one edge, less than both footprints together
    two = p.step(np.union1d(a, _disc(pos, frac((1.0 + 0.35 + 0.2 + 0.78, 2.0)), 0.2)))
    # the last pass runs from every lethal (both clusters are affected) and settles what the full wave settles; the
    # first pass, from the disc alone, comes on top
    assert two["settled"] > p.ref["settled"], (two["settled"], p.ref["settled"])
    p.close()


@pytest.mark.gpu
def test_repair_whole_map_switch(api, oracle_mod):
    """when most of the old footprint is in affected clusters the call runs the whole-map wave itself: the same bits and
    changed set, the full wave's work, and whole-map labels for mnb_inflation_vector_map; an unchanged set runs no wave
    and keeps those labels; a small change afterwards takes the local path again and keeps the field valid"""
    pos, faces = mesh_case(40, True)
    p = Pair(api, oracle_mod, pos, faces, 0.4, field=False)
    centres = [(x, y) for x in (0.15, 0.5, 0.85) for y in (0.15, 0.5, 0.85)]     # footprints 1.3 m wide, 1.37 m apart
    disc_list = lambda dx: [_disc(pos, (x + dx, y), 0.1) for x, y in centres]
    discs = lambda dx: np.unique(np.concatenate(disc_list(dx))).astype(np.uint32)
    p.step(discs(0.0))
    p.step(discs(0.02))                                          # every cluster moves
    moved = p.step(discs(0.04))
    assert moved["settled"] == p.ref["settled"] and moved["rounds"] == p.ref["rounds"]
    assert _same(p.rep.vectorMap(), p.full.vectorMap())
    again = p.step(discs(0.04))
    assert again["changed"].size == 0 and again["settled"] == 0
    assert _same(p.rep.vectorMap(), p.full.vectorMap())
    one = disc_list(0.04)
    one[-1] = _disc(pos, (0.85 + 0.06, 0.85), 0.1)                # one cluster of nine moves
    local = p.step(np.unique(np.concatenate(one)).astype(np.uint32))
    assert 0 < local["settled"] < p.ref["settled"]
    # the field became valid after the whole-map waves, so the local repair kept it up to date on its region
    assert _same(p.rep.vectorMap(), p.full.vectorMap())
    p.close()


@pytest.mark.gpu
def test_repair_invalid_flip(api, oracle_mod):
    """an invalid flag flips inside a cluster that no lethal change touches, and flips back"""
    pos, faces = mesh_case(36, False)
    V = pos.shape[0]
    p = Pair(api, oracle_mod, pos, faces, 0.5)
    a, b = _disc(pos, (0.25, 0.5), 0.2), _disc(pos, (0.75, 0.5), 0.2)
    le = np.union1d(a, b).astype(np.uint32)
    inv = np.zeros(V, np.uint8)
    p.step(le, inv)
    ring = np.setdiff1d(_disc(pos, (0.75, 0.5), 0.32), b)
    inv2 = inv.copy(); inv2[ring[::3]] = 1
    r = p.step(le, inv2)
    assert r["changed"].size > 0
    assert r["settled"] < V // 2
    p.step(le, inv)
    p.step(le, None)                                             # NULL mask == all valid: nothing changes
    p.close()


@pytest.mark.gpu
def test_repair_params_and_first_call(api, oracle_mod):
    """no previous result, then other params: whole-map waves, changed sets against the previous riskiness"""
    pos, faces = mesh_case(30, True)
    p = Pair(api, oracle_mod, pos, faces, 0.4)
    le = _disc(pos, (0.5, 0.5), 0.3)
    p.step(le)
    p.step(np.union1d(le, _disc(pos, (0.1, 0.9), 0.1)))
    for layer in (p.rep, p.full):
        layer.config.inflation_radius = 0.55
    p.radius = 0.55
    p.step(le)
    p.step(np.union1d(le, _disc(pos, (0.9, 0.1), 0.1)))
    p.close()


@pytest.mark.gpu
def test_repair_interleaved(api, oracle_mod):
    """planner calls (CVP, Dijkstra batch) between steps and full calls mixed into a chain of repairs"""
    pos, faces = mesh_case(36, True)
    p = Pair(api, oracle_mod, pos, faces, 0.4)
    vc = np.zeros(p.V, np.float32)
    p.rmap.setCosts(vc, p.rmap.edgeDistances())
    v, f, sp = centre_seed(pos, faces, (0.5, 0.5))
    cvp = api.CVPMeshPlanner(p.rmap)
    dij = api.DijkstraMeshPlanner(p.rmap)
    static = _disc(pos, (0.2, 0.2), 0.25)
    plan = lambda: (cvp.waveFrontPropagation(f, sp), dij.dijkstraBatch(np.array([3, 500], np.uint32)))
    p.step(static)
    plan()
    for k, (x, full) in enumerate([(0.5, False), (0.55, False), (0.6, True), (0.65, False), (0.7, False), (0.75, True)]):
        p.step(np.union1d(static, _disc(pos, (x, 0.6), 0.2)), repair=not full)
        plan()
        assert (cvp.waveFrontPropagation(f, sp)["outcome"]) == 0
    # a field that was not valid before a repair is not available after it
    q = Pair(api, oracle_mod, pos, faces, 0.4, oracle=False, field=False)
    q.step(static); q.step(np.union1d(static, _disc(pos, (0.6, 0.6), 0.2)))
    with pytest.raises(RuntimeError):
        q.rep.vectorMap()
    p.close(); q.close()


@pytest.mark.gpu
def test_repair_pointer_modes_and_errors(api, oracle_mod):
    """device pointers give the bytes of host pointers; argument errors write nothing and keep the resident result"""
    pos, faces = mesh_case(30, True)
    p = Pair(api, oracle_mod, pos, faces, 0.4, field=False)
    V = p.V
    a = _disc(pos, (0.3, 0.3), 0.2)
    p.step(a)
    L, ctx, cfg = p.rmap.L, p.rmap._ctx, C.byref(p.rep.config)
    le = np.union1d(a, _disc(pos, (0.7, 0.7), 0.2)).astype(np.uint32)
    dist = np.full(V, 7.0, np.float32); cost = dist.copy(); chg = np.full(V, 9, np.uint32); n = C.c_uint32(123)
    P = lambda x: x.ctypes.data
    assert L.mnb_inflation_repair(ctx, None, 5, None, cfg, P(dist), P(cost), P(chg), C.byref(n)) == -1
    assert L.mnb_inflation_repair(ctx, P(le), le.size, None, None, P(dist), P(cost), P(chg), C.byref(n)) == -1
    assert L.mnb_inflation_repair(ctx, P(le), le.size, None, cfg, P(dist), P(cost), P(chg), None) == -1
    assert (dist == 7.0).all() and (cost == 7.0).all() and (chg == 9).all() and n.value == 123
    ref = p.full.onInputChanged(le)
    exp = _changed(ref["cost"], p.prev)
    on_gpu = not hasattr(L, "mnb_emu_switch")
    if on_gpu:
        import torch
        t_le = torch.from_numpy(le.view(np.int32)).cuda()
        t_d = torch.empty(V, dtype=torch.float32, device="cuda"); t_c = torch.empty_like(t_d)
        t_ch = torch.empty(V, dtype=torch.int32, device="cuda")
        ptrs = (t_le.data_ptr(), t_d.data_ptr(), t_c.data_ptr(), t_ch.data_ptr())
        back = lambda: (t_d.cpu().numpy(), t_c.cpu().numpy(), t_ch.cpu().numpy().view(np.uint32))
    else:                        # the interpreter runs the leg with host pointers
        ptrs = (P(le), P(dist), P(cost), P(chg))
        back = lambda: (dist, cost, chg)
    p.rmap.use_device_pointers(on_gpu)
    try:
        assert L.mnb_inflation_repair(ctx, ptrs[0], le.size, None, cfg, ptrs[1], ptrs[2], ptrs[3], C.byref(n)) == 0
        if on_gpu:
            torch.cuda.synchronize()
    finally:
        p.rmap.use_device_pointers(False)
    gd, gc, gch = back()
    assert _same(gd, ref["dist"]) and _same(gc, ref["cost"]) and np.array_equal(gch[:n.value], exp)
    # NULL outputs: only the count
    le2 = a
    assert L.mnb_inflation_repair(ctx, P(le2), le2.size, None, cfg, None, None, None, C.byref(n)) == 0
    ref2 = p.full.onInputChanged(le2)
    assert n.value == _changed(ref2["cost"], ref["cost"]).size
    p.prev = ref2["cost"]
    p.step(le)                                                   # the resident result followed every call
    p.close()


@pytest.mark.gpu
def test_repair_pipeline(api, oracle_mod):
    """obstacle layer -> inflation repair -> max combination on the changed set -> layerChanged -> Dijkstra field repair:
    the rows are bit-identical to a fresh batch on a fully re-installed map"""
    pos, faces = mesh_case(40, True)
    V = pos.shape[0]
    mm = api.MeshMap(pos, faces)
    ed = mm.edgeDistances()
    rng = np.random.default_rng(4)
    static = (rng.random(V) * 0.3).astype(np.float32)
    factor = 1.0
    O = oracle_mod
    om = O.OracleMesh(pos, faces)
    mm.setCosts(static.copy(), om.edge_weights(static, ed, factor))
    obst = api.ObstacleLayer(mm, robot_height=1.0)
    infl = api.InflationLayer(mm)
    pl = api.DijkstraMeshPlanner(mm, cost_limit=0.95)
    seeds = np.array([17, 800, 1500], np.uint32)
    rows = pl.dijkstraBatch(seeds)
    final = static.copy()
    first = True
    for cyc, centre in enumerate([(0.3, 0.3), (0.35, 0.3), (0.7, 0.6), (0.7, 0.65)]):
        d = _disc(pos, centre, 0.2)
        pts = pos[d] + np.array([0, 0, 0.3], np.float32)
        ob = obst.processPointCloud(pts)
        got = infl.onInputChanged(ob["lethals"]) if first else infl.repairInflation(ob["lethals"])
        first = False
        mm.maxCombinationUpdate([static, got["cost"]], [0.0, 0.0], None, got["changed"], final, None)
        mm.layerChanged(got["changed"], final, factor, by_vertex=True)
        r = pl.dijkstraBatchRepair(seeds, got["changed"], rows["dist"], rows["pred"])
        assert r["outcome"] == 0
        fresh_map = api.MeshMap(pos, faces)
        fresh_map.setCosts(final.copy(), om.edge_weights(final, ed, factor))
        ref = api.DijkstraMeshPlanner(fresh_map, cost_limit=0.95).dijkstraBatch(seeds)
        fresh_map.close()
        assert _same(rows["dist"], ref["dist"]) and (rows["pred"] == ref["pred"]).all(), f"cycle {cyc}"
    mm.close()


@pytest.mark.gpu
def test_repair_work_large_mesh(api, oracle_mod):
    """1 M-vertex terrain with layer lethals and about 200 discs: moving one disc settles under 5 % of the full wave"""
    pos, faces = mesh_case(1000, True)
    V = pos.shape[0]
    layer = np.union1d(_disc(pos, (0.5, 0.5), 3.0), np.where(pos[:, 0] <= pos[:, 0].min() + 0.02)[0]).astype(np.uint32)
    discs = disc_lethals(pos, 200, 0.25, seed=21)
    p = Pair(api, oracle_mod, pos, faces, 0.4, oracle=False, field=False)
    base = np.union1d(layer, discs).astype(np.uint32)
    full = p.step(base, repair=False)
    moved = np.union1d(base, _disc(pos, (0.12, 0.9), 0.25)).astype(np.uint32)
    p.step(moved)
    moved2 = np.union1d(base, _disc(pos, (0.125, 0.9), 0.25)).astype(np.uint32)
    r = p.step(moved2)
    print(f"settled {r['settled']} of {full['settled']}, rounds {r['rounds']} of {full['rounds']}, changed {r['changed'].size}")
    assert r["settled"] < 0.05 * full["settled"]
    p.close()


def test_oracle_inflation_decomposes_into_clusters(oracle_mod):
    """the premise of the repair: the oracle's inflation (distances and vector map) from a lethal set S is the union of
    its inflations from the lethals of each cluster of S's footprint alone"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    O = oracle_mod
    cases = [(mesh_case(30, True), None, 0.4), (synth.grid_mesh(28, 28, jitter=0.0, terrain=False), None, 0.5),
             (delaunay_mesh(700, seed=8, extent=3.0), 0.05, 0.4), (mesh_case(26, False, seed=3), 0.03, 0.6)]
    rng = np.random.default_rng(17)
    n_clusters = 0
    for (pos, faces), p_inv, radius in cases:
        V = pos.shape[0]
        om = O.OracleMesh(pos, faces)
        ed = om.edge_distances()
        inv = (rng.random(V) < p_inv).astype(np.uint8) if p_inv else None
        corners = [(0.2, 0.2), (0.8, 0.2), (0.2, 0.8), (0.8, 0.8), (0.5, 0.5)]
        le = np.unique(np.concatenate([_disc(pos, np.asarray(c) + 0.04 * rng.random(2), 0.05 + 0.1 * rng.random())
                                       for c in corners])).astype(np.uint32)
        ref = om.inflation(ed, le, invalid=inv, inflation_radius=radius, with_vectors=True)
        foot = np.isfinite(ref["dist"])
        f = faces.astype(np.int64)
        pairs = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [0, 2]]])
        pairs = pairs[foot[pairs[:, 0]] & foot[pairs[:, 1]]]
        g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(V, V))
        n_comp, comp = connected_components(g, directed=False)
        clusters = [c for c in np.unique(comp[foot])]
        n_clusters += len(clusters)
        for c in clusters:
            mask = foot & (comp == c)
            sub = om.inflation(ed, le[mask[le]], invalid=inv, inflation_radius=radius, with_vectors=True)
            assert np.array_equal(np.isfinite(sub["dist"]), mask)
            assert _same(sub["dist"][mask], ref["dist"][mask])
            assert _same(sub["vectors"][mask], ref["vectors"][mask])
            assert (sub["vectors"][~mask] == 0).all()
    assert n_clusters >= 2 * len(cases)


def test_inflation_repair_on_the_cpu_interpreter():
    """the GPU tests above (minus the 1 M-vertex one) with the kernels compiled by g++ against tests/emu, on 4 emulated
    SMs, in the default warp order and in a randomised one"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    for extra in ({}, {"MNB_EMU_SHUFFLE": "3"}):
        env = dict(os.environ, MNB_EMU_SMS="4", **extra)
        r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider", "-k", "not large_mesh"],
                           cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
        tail = (r.stdout + r.stderr)[-3000:]
        assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"{extra}:\n{tail}"
