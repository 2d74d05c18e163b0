"""Cost matrices (mnb_dijkstra_matrix / mnb_cvp_matrix, DijkstraMeshPlanner.costMatrix / CVPMeshPlanner.costMatrix):
entry [k, j] against the gathered rows of mnb_dijkstra_batch / mnb_cvp_batch and against the oracle's
DijkstraMeshPlanner::dijkstra / CVPMeshPlanner::waveFrontPropagation at the target vertex, bit for bit as uint32.  A
wave stops once its targets have settled; the statistics show the work saved.  The GPU tests run with -m gpu on an
H100; the last test replays them on the CPU interpreter of the kernels (tests/emu)."""
import ctypes as C
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from tests.util import centre_seed, mesh_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ("dijkstra", "cvp")


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def _map(api, oracle_mod, pos, faces, costs=None, factor=0.0, invalid=None):
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    vc = np.zeros(om.V, np.float32) if costs is None else np.asarray(costs, np.float32)
    w = om.edge_weights(vc, om.edge_distances(), factor)
    mm.setCosts(vc, w, invalid)
    return om, mm, vc, w


class Case:
    """one map and one planner kind; seeds are given as vertices (CVP: the first face of the vertex, at its centroid)"""

    def __init__(self, api, om, mm, vc, w, pos, faces, kind, invalid=None, cost_limit=1.0):
        self.api, self.om, self.mm, self.vc, self.w, self.kind = api, om, mm, vc, w, kind
        self.pos, self.faces, self.invalid, self.cost_limit = pos, np.asarray(faces, np.uint32), invalid, cost_limit
        first = np.empty(om.V, np.int64)
        first[self.faces.ravel()[::-1]] = np.repeat(np.arange(len(self.faces)), 3)[::-1]
        self.first_face = first
        if kind == "dijkstra":
            self.pl = api.DijkstraMeshPlanner(mm, cost_limit=cost_limit)
        else:
            self.pl = api.CVPMeshPlanner(mm, cost_limit=cost_limit)

    def goals(self, seeds):
        sfs = self.first_face[np.asarray(seeds, np.int64)].astype(np.uint32)
        return sfs, np.stack([self.pos[self.faces[f]].mean(0) for f in sfs]).astype(np.float32).reshape(-1, 3)

    def seed_vertices(self, s):
        """the vertices a wave seeded at vertex s starts from"""
        return [int(s)] if self.kind == "dijkstra" else [int(x) for x in self.faces[self.first_face[int(s)]]]

    def matrix(self, seeds, targets):
        if self.kind == "dijkstra":
            return self.pl.costMatrix(seeds, targets)
        return self.pl.costMatrix(*self.goals(seeds), targets)

    def rows(self, seeds):
        if self.kind == "dijkstra":
            return self.pl.dijkstraBatch(seeds, want_pred=False)
        return self.pl.waveFrontPropagationBatch(*self.goals(seeds))

    def raw(self, seeds, targets, fill=7.0, seeds_ptr=True, targets_ptr=True, out_ptr=True, pos_ptr=True):
        """the C entry point in host-pointer mode, output pre-filled"""
        sv = np.ascontiguousarray(seeds, dtype=np.uint32); tv = np.ascontiguousarray(targets, dtype=np.uint32)
        out = np.full((max(sv.size, 1), max(tv.size, 1)), fill, np.float32)
        p = lambda a, on: a.ctypes.data_as(C.c_void_p) if on else None
        L, ctx = self.mm.L, self.mm._ctx
        if self.kind == "dijkstra":
            rc = L.mnb_dijkstra_matrix(ctx, sv.size, p(sv, seeds_ptr), tv.size, p(tv, targets_ptr), self.cost_limit, p(out, out_ptr))
        else:                          # a seed vertex >= V becomes the seed face F
            F = len(self.faces)
            sfs = np.array([self.first_face[s] if s < self.om.V else F for s in sv], np.uint32)
            sps = np.array([self.pos[self.faces[f]].mean(0) if f < F else np.zeros(3) for f in sfs], np.float32).reshape(-1, 3)
            rc = L.mnb_cvp_matrix(ctx, sv.size, p(sfs, seeds_ptr), p(sps, pos_ptr), tv.size, p(tv, targets_ptr), self.cost_limit,
                                  p(out, out_ptr))
        return rc, out

    def oracle_entries(self, seeds, targets):
        out = []
        sfs, sps = self.goals(seeds)
        for k, s in enumerate(seeds):
            if self.kind == "dijkstra":
                d = self.om.dijkstra(self.w, self.vc, int(s), invalid=self.invalid, cost_limit=self.cost_limit)["dist"]
            else:
                d = self.om.cvp(self.w, self.vc, int(sfs[k]), sps[k], invalid=self.invalid, cost_limit=self.cost_limit)["dist"]
            out.append(np.asarray(d, np.float32)[np.asarray(targets, np.int64)])
        return np.stack(out)

    def check(self, seeds, targets, oracle=True):
        """matrix == gathered batch rows (and the oracle); returns both results"""
        got = self.matrix(seeds, targets)
        ref = self.rows(seeds)
        assert got["outcome"] == 0 and ref["outcome"] == 0
        assert got["cost"].shape == (len(seeds), len(targets))
        assert _same(got["cost"], ref["dist"][:, np.asarray(targets, np.int64)]), self.kind
        if oracle:
            assert _same(got["cost"], self.oracle_entries(seeds, targets)), self.kind
        return got, ref


def _wall_costs(pos, rng):
    """cost regions over the cost limit, and a +inf wall that leaves the far side of the map unreached"""
    c = np.where(rng.random(pos.shape[0]) < 0.05, 1.5, rng.random(pos.shape[0]) * 0.8).astype(np.float32)
    c[(pos[:, 0] > 3.0) & (pos[:, 0] < 3.4)] = np.inf
    return c


def _walled_case(api, oracle_mod, kind, factor, n=50, seed=11):
    rng = np.random.default_rng(seed)
    pos, faces = mesh_case(n, True)
    costs = _wall_costs(pos, rng)
    invalid = (rng.random(pos.shape[0]) < 0.01).astype(np.uint8)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, costs, factor, invalid)
    return Case(api, om, mm, vc, w, pos, faces, kind, invalid=invalid), rng


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_parity(api, oracle_mod, kind, factor):
    """cost walls, an over-limit region, invalid vertices; targets include a seed, an invalid and an over-cost vertex and
    duplicates"""
    cs, rng = _walled_case(api, oracle_mod, kind, factor)
    V = cs.om.V
    over = np.where((cs.vc > 1.0) & np.isfinite(cs.vc) & (cs.invalid == 0))[0]
    inv = np.where(cs.invalid != 0)[0]
    seeds = rng.choice(np.setdiff1d(np.arange(V), np.concatenate([over, inv])), 10, replace=False).astype(np.uint32)
    targets = np.concatenate([rng.choice(V, 30, replace=False), cs.seed_vertices(seeds[0]), inv[:2], over[:3],
                              [seeds[3], seeds[3]]]).astype(np.uint32)
    targets = np.concatenate([targets, targets[:5]])
    got, ref = cs.check(seeds, targets)
    cost = got["cost"]
    assert np.isinf(cost).any() and np.isfinite(cost).any()
    # entries of targets that are not one of the goal's own seed vertices
    other = np.stack([~np.isin(targets, cs.seed_vertices(s)) for s in seeds])
    assert np.isinf(cost[other & np.isin(targets, inv)[None, :]]).all()          # invalid: never a candidate
    over_t = other & np.isin(targets, over)[None, :]
    if kind == "cvp":
        assert np.isinf(cost[over_t]).all()                                     # over the cost limit: never a CVP candidate
    else:
        assert np.isfinite(cost[over_t]).any()                                  # a Dijkstra label, but no expansion
    assert np.isfinite(cost[0, np.isin(targets, cs.seed_vertices(seeds[0]))]).all()
    assert got["settled"] <= ref["settled"] and got["kernel_launches"] == 1
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_edge_targets(api, oracle_mod, kind):
    """m = 1; every vertex a target (the matrix is the full rows); all targets done before the first round; a target in
    another component (the wave runs in full)"""
    rng = np.random.default_rng(5)
    pos, faces = mesh_case(40, True)
    costs = np.where(rng.random(pos.shape[0]) < 0.1, 1.5, 0.3).astype(np.float32)
    invalid = (rng.random(pos.shape[0]) < 0.02).astype(np.uint8)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, costs, 1.0, invalid)
    cs = Case(api, om, mm, vc, w, pos, faces, kind, invalid=invalid)
    v = centre_seed(pos, faces)[0]
    far = centre_seed(pos, faces, (0.9, 0.85))[0]
    cs.check([v], [far])
    seeds = np.array([v, far, 17], np.uint32)
    got, ref = cs.check(seeds, np.arange(om.V, dtype=np.uint32))
    assert _same(got["cost"], ref["dist"]) and got["settled"] == ref["settled"]
    # every target done at init: the seed's own vertices, invalid vertices (and for CVP over-cost ones): no round runs
    never = np.where(invalid)[0][:3]
    if kind == "cvp":
        never = np.concatenate([never, np.where((vc > 1.0) & (invalid == 0))[0][:3]])
    never = [int(x) for x in never if int(x) not in cs.seed_vertices(v)]
    got, _ = cs.check([v], cs.seed_vertices(v) + never)
    assert got["rounds"] == 0 and got["settled"] == 0, (got["rounds"], got["settled"])
    ns = len(cs.seed_vertices(v))
    assert np.isfinite(got["cost"][0, :ns]).all() and np.isinf(got["cost"][0, ns:]).all()
    mm.close()
    # two components: a target in the other one is never reached, so the wave settles everything it can reach
    pos1, faces1 = mesh_case(20, False)
    pos = np.concatenate([pos1, pos1 + np.array([10.0, 0, 0], np.float32)])
    faces = np.concatenate([faces1, faces1 + len(pos1)]).astype(np.uint32)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces)
    cs = Case(api, om, mm, vc, w, pos, faces, kind)
    n1 = len(pos1)
    seeds = np.array([5, n1 + 7, 5], np.uint32)
    got, ref = cs.check(seeds, [6, n1 + 3, n1 + 3])
    assert got["settled"] == ref["settled"] and np.isinf(got["cost"][0, 1]) and np.isinf(got["cost"][1, 0])
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_early_stop(api, oracle_mod, kind):
    """seeds and targets inside a small window of a 90 x 90 terrain: exact entries for a fraction of the settled vertices"""
    rng = np.random.default_rng(9)
    pos, faces = mesh_case(90, True)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, (rng.random(8100) * 0.5).astype(np.float32), 1.0)
    cs = Case(api, om, mm, vc, w, pos, faces, kind)
    i, j = np.meshgrid(np.arange(40, 50), np.arange(40, 50))
    window = (j * 90 + i).ravel()
    seeds = rng.choice(window, 6, replace=False).astype(np.uint32)
    targets = rng.choice(window, 12, replace=False).astype(np.uint32)
    got, ref = cs.check(seeds, targets)
    ratio = got["settled"] / ref["settled"]
    print(f"{kind}: settled {got['settled']} of {ref['settled']} ({ratio:.3f}), rounds {got['rounds']} of {ref['rounds']}")
    assert ratio < 0.2, ratio
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour"])
def test_cost_matrix_cvp_fuzz_fixtures(api, oracle_mod, name):
    """deep cascades, cost-limit walls and seeds that pop after their neighbours, at two launch shapes"""
    d = np.load(os.path.join(ROOT, "tests", "golden", f"fuzz_{name}.npz"))
    inv = d["inv"] if d["inv"].size else None
    pos, faces, vc, w, sf, sp, cl = d["pos"], d["faces"], d["vc"], d["w"], int(d["sf"]), d["sp"], float(d["cl"])
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w, inv)
    pl = api.CVPMeshPlanner(mm, cost_limit=cl)
    rng = np.random.default_rng(5)
    sfs = np.concatenate([[sf], rng.integers(0, om.F, 3)]).astype(np.uint32)
    sps = np.stack([pos[faces[f]].mean(0) for f in sfs]).astype(np.float32)
    sps[0] = sp
    targets = np.concatenate([rng.choice(om.V, min(40, om.V), replace=False), faces[sf]]).astype(np.uint32)
    refs = np.stack([np.asarray(om.cvp(w, vc, int(sfs[k]), sps[k], invalid=inv, cost_limit=cl)["dist"], np.float32)[targets]
                     for k in range(len(sfs))])
    for cluster, delta in ((1, 0.3), (4, 0.05)):
        mm.set_tuning(delta, cluster, 0)
        got = pl.costMatrix(sfs, sps, targets)
        rows = pl.waveFrontPropagationBatch(sfs, sps)
        assert got["outcome"] == 0
        assert _same(got["cost"], rows["dist"][:, targets]) and _same(got["cost"], refs), (cluster, delta)
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_shapes(api, oracle_mod, kind):
    """1, 3 and 600 seeds; cluster sizes 1, 2, 4, 8 and two band widths give the same entries"""
    rng = np.random.default_rng(3)
    pos, faces = mesh_case(40, True)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, (rng.random(1600) * 0.8).astype(np.float32), 1.0)
    cs = Case(api, om, mm, vc, w, pos, faces, kind)
    seeds = rng.choice(om.V, 3, replace=False).astype(np.uint32)
    targets = rng.choice(om.V, 25, replace=False).astype(np.uint32)
    for n in (1, 3):
        base, _ = cs.check(seeds[:n], targets)
    for cluster in (1, 2, 4, 8):
        for delta in (0.02, 1.0):
            mm.set_tuning(delta, cluster, 0)
            got = cs.matrix(seeds, targets)
            assert got["outcome"] == 0 and _same(got["cost"], base["cost"]), (cluster, delta)
    mm.close()
    pos, faces = mesh_case(20, True)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, (rng.random(400) * 0.8).astype(np.float32), 1.0)
    cs = Case(api, om, mm, vc, w, pos, faces, kind)
    seeds = rng.integers(0, om.V, 600).astype(np.uint32)
    targets = rng.choice(om.V, 7, replace=False).astype(np.uint32)
    got, _ = cs.check(seeds, targets, oracle=False)
    uniq, first = np.unique(seeds, return_index=True)
    ref = cs.oracle_entries(uniq, targets)
    assert _same(got["cost"][first], ref)
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_pointer_modes(api, oracle_mod, kind):
    """device pointers give the same bytes as host pointers"""
    rng = np.random.default_rng(8)
    pos, faces = mesh_case(30, True)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, (rng.random(900) * 0.8).astype(np.float32), 1.0)
    cs = Case(api, om, mm, vc, w, pos, faces, kind)
    seeds = rng.choice(om.V, 5, replace=False).astype(np.uint32)
    targets = rng.choice(om.V, 9, replace=False).astype(np.uint32)
    host, _ = cs.check(seeds, targets)
    # decided by the loaded library: the CPU interpreter (it exports its fiber switch) cannot dereference device pointers
    on_gpu = not hasattr(mm.L, "mnb_emu_switch")
    if on_gpu:
        import torch
        buf = torch.full((seeds.size, targets.size), 7.0, dtype=torch.float32, device="cuda")
        ptr = buf.data_ptr(); back = lambda: buf.cpu().numpy()
    else:
        buf = np.full((seeds.size, targets.size), 7.0, np.float32)
        ptr = buf.ctypes.data; back = lambda: buf
    mm.use_device_pointers(True)
    try:
        if kind == "dijkstra":
            assert mm.dijkstra_matrix_dev(seeds, targets, 1.0, ptr) == 0
        else:
            sfs, sps = cs.goals(seeds)
            assert mm.cvp_matrix_dev(sfs, sps, targets, 1.0, ptr) == 0
        if on_gpu:
            torch.cuda.synchronize()
        assert _same(back(), host["cost"])
    finally:
        mm.use_device_pointers(False)
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_arguments(api, oracle_mod, kind):
    """no costs -> MNB_E_STATE (-3); n == 0, m == 0 or a NULL array -> MNB_E_ARG (-1); a seed out of range ->
    INVALID_START (52); a target >= V -> INVALID_GOAL (53); nothing written in any of these"""
    pos, faces = mesh_case(20, True)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    cs = Case(api, om, mm, np.zeros(om.V, np.float32), om.edge_distances(), pos, faces, kind)
    untouched = lambda out: (out == 7.0).all()
    rc, out = cs.raw([3, 4], [5, 6])
    assert rc == -3 and untouched(out)
    mm.setCosts(cs.vc, cs.w)
    for kw in (dict(seeds_ptr=False), dict(targets_ptr=False), dict(out_ptr=False)) + ((dict(pos_ptr=False),) if kind == "cvp" else ()):
        rc, out = cs.raw([3, 4], [5, 6], **kw)
        assert rc == -1 and untouched(out), kw
    rc, out = cs.raw([], [5, 6])
    assert rc == -1 and untouched(out)
    rc, out = cs.raw([3, 4], [])
    assert rc == -1 and untouched(out)
    rc, out = cs.raw([3, om.V, 4], [5, 6])                      # CVP: the seed face becomes F
    assert rc == 52 and untouched(out)
    rc, out = cs.raw([3, 4], [5, om.V, 6])
    assert rc == 53 and untouched(out)
    rc, out = cs.raw([3, 4], [5, 6])
    assert rc == 0 and _same(out, cs.oracle_entries([3, 4], [5, 6]))
    mm.close()


@pytest.mark.gpu
def test_cost_matrix_state(api, oracle_mod):
    """a Dijkstra matrix leaves the last mnb_cvp's back-tracking path, mnb_vector_map(pred = NULL) and the last inflation's
    vector map alone; a CVP matrix leaves the last mnb_cvp's outputs alone; after layerChanged both use the new weights"""
    rng = np.random.default_rng(21)
    pos, faces = mesh_case(50, True)
    costs = (0.45 + 0.45 * np.sin(3.0 * pos[:, 0])).astype(np.float32)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces, costs, 1.0)
    dcs = Case(api, om, mm, vc, w, pos, faces, "dijkstra")
    ccs = Case(api, om, mm, vc, w, pos, faces, "cvp")
    seeds = rng.choice(om.V, 6, replace=False).astype(np.uint32)
    targets = rng.choice(om.V, 10, replace=False).astype(np.uint32)
    sv, sf, sp = centre_seed(pos, faces, (0.2, 0.25))
    rv, rf, rp = centre_seed(pos, faces, (0.8, 0.7))
    out = np.empty((om.V, 3), np.float32)
    vec = lambda: (mm.L.mnb_vector_map(mm._ctx, None, None, None, out.ctypes.data_as(C.c_void_p)), out.copy())[1]
    cpl = ccs.pl
    infl = api.InflationLayer(mm)
    assert cpl.waveFrontPropagation(sf, sp, rf)["outcome"] == 0
    bt0 = cpl.backtrack(rp, rf); vm0 = vec()
    infl.waveCostInflation(np.array([sv, rv], np.uint32))
    iv0 = infl.vectorMap()
    assert dcs.matrix(seeds, targets)["outcome"] == 0
    bt1 = cpl.backtrack(rp, rf); vm1 = vec(); iv1 = infl.vectorMap()
    assert bt0["outcome"] == bt1["outcome"] == 0 and len(bt0["positions"]) > 5
    assert _same(bt0["positions"], bt1["positions"]) and (bt0["faces"] == bt1["faces"]).all() and _same(vm0, vm1)
    assert _same(iv0, iv1)
    assert cpl.waveFrontPropagation(sf, sp, rf)["outcome"] == 0
    assert ccs.matrix(seeds, targets)["outcome"] == 0
    bt2 = cpl.backtrack(rp, rf); vm2 = vec()
    assert _same(bt0["positions"], bt2["positions"]) and (bt0["faces"] == bt2["faces"]).all() and _same(vm0, vm2)
    changed = np.unique(rng.choice(om.V, 300, replace=False)).astype(np.uint32)
    mm.layerChanged(changed, (rng.random(changed.size) * 0.9).astype(np.float32), 1.0)
    vc2, w2 = mm.costs()
    assert (w2 != w).any()
    for cs in (dcs, ccs):
        cs.vc, cs.w = vc2, w2
        cs.check(seeds, targets)
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cost_matrix_cancel(api, oracle_mod, kind):
    """mnb_cancel from another thread -> CANCELED (51); the persistent groups take no new goals; the next call is exact"""
    pos, faces = mesh_case(120 if kind == "dijkstra" else 60, True)      # as in the batch calls' cancel tests
    om, mm, vc, w = _map(api, oracle_mod, pos, faces)
    mm.set_tuning(0.005, 1, 0)         # narrow band: many rounds per wavefront
    cs = Case(api, om, mm, vc, w, pos, faces, kind)
    targets = np.array([0, om.V - 1], np.uint32)     # opposite corners: every wave runs nearly in full
    rng = np.random.default_rng(2)
    n = 8
    while True:                        # grow the batch until it takes long enough for the cancel to land inside it
        seeds = rng.integers(0, om.V, n).astype(np.uint32)
        cs.matrix(seeds, targets)      # a first call at a size grows the workspace: not part of the time the cancel aims at
        t0 = time.perf_counter(); full = cs.matrix(seeds, targets); t_full = time.perf_counter() - t0
        assert full["outcome"] == 0
        if t_full > 0.2 or n >= 16384:
            break
        n *= 4
    assert t_full > 0.05, t_full
    outcomes = []

    def run():
        t1 = time.perf_counter(); o = cs.matrix(seeds, targets)["outcome"]; outcomes.append((o, time.perf_counter() - t1))
    t = threading.Thread(target=run)
    t.start(); time.sleep(0.25 * t_full); mm.cancel(); t.join()
    assert outcomes[0][0] == 51, outcomes
    assert outcomes[0][1] < 0.85 * t_full, (outcomes, t_full)
    got = cs.matrix(seeds[:2], targets)
    assert got["outcome"] == 0 and _same(got["cost"], full["cost"][:2])
    mm.close()


@pytest.mark.gpu
def test_cost_matrix_large_mesh(api, oracle_mod):
    """1 M-vertex terrain, 64 seeds x 256 targets, sampled rows against the oracle"""
    from mesh_navigation_b200 import synth
    pos, faces = mesh_case(1000, True)
    om, mm, vc, w = _map(api, oracle_mod, pos, faces)
    seeds = synth.batch_goal_vertices(om.V, 64, seed=1234).astype(np.uint32)
    targets = synth.batch_goal_vertices(om.V, 256, seed=77).astype(np.uint32)
    for kind in KINDS:
        cs = Case(api, om, mm, vc, w, pos, faces, kind)
        got = cs.matrix(seeds, targets)
        assert got["outcome"] == 0 and np.isfinite(got["cost"]).all()
        rows = [0, 21, 42, 63]
        assert _same(got["cost"][rows], cs.oracle_entries(seeds[rows], targets)), kind
    mm.close()


def test_cost_matrix_on_the_cpu_interpreter():
    """the GPU tests above (minus the 1 M-vertex one) with the kernels compiled by g++ against tests/emu, on 4 emulated
    SMs, in the default warp order and in a randomised one (the check on the done flag's round discipline)"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    for extra in ({}, {"MNB_EMU_SHUFFLE": "3"}):
        env = dict(os.environ, MNB_EMU_SMS="4", **extra)
        r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider", "-k", "not large_mesh"],
                           cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
        tail = (r.stdout + r.stderr)[-3000:]
        assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"{extra}:\n{tail}"
