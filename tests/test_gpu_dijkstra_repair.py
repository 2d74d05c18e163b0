"""Dijkstra field repair (mnb_dijkstra_batch_repair / DijkstraMeshPlanner.dijkstraBatchRepair): rows of
mnb_dijkstra_batch on costs A, an mnb_update_vertex_costs to costs B, the repair -- then every row bit for bit (as uint32,
predecessors included) against a fresh mnb_dijkstra_batch on B, and on the small meshes against the oracle's
DijkstraMeshPlanner::dijkstra on B.  The GPU tests run with -m gpu on an H100; the last test replays them on the CPU
interpreter of the kernels (tests/emu)."""
import ctypes as C
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from mesh_navigation_b200 import synth
from tests.util import centre_seed, delaunay_mesh, mesh_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def _mesh(kind):
    if kind == "terrain":
        return mesh_case(36, True)
    if kind == "planar":
        return mesh_case(36, False)
    if kind == "exact_ties":                         # unjittered planar grid: many equal sums, the predecessor tie rule
        return synth.grid_mesh(34, 34, jitter=0.0, terrain=False)
    if kind == "delaunay":
        return delaunay_mesh(1100, seed=5, extent=3.6)
    raise ValueError(kind)


class Case:
    """one map, its seeds and the rows of the last fresh batch or repair"""

    def __init__(self, api, oracle_mod, pos, faces, costs, factor=1.0, invalid=None, cost_limit=1.0, oracle=True):
        self.api, self.pos, self.faces, self.factor, self.invalid, self.cost_limit = api, pos, faces, factor, invalid, cost_limit
        self.om = oracle_mod.OracleMesh(pos, faces)
        self.mm = api.MeshMap(pos, faces)
        self.ed = self.om.edge_distances()
        vc = np.asarray(costs, np.float32)
        self.mm.setCosts(vc, self.om.edge_weights(vc, self.ed, factor), invalid)
        self.pl = api.DijkstraMeshPlanner(self.mm, cost_limit=cost_limit)
        self.oracle = oracle
        self.vc = vc.copy()

    def fresh(self, seeds):
        r = self.pl.dijkstraBatch(seeds)
        assert r["outcome"] == 0
        return r

    def update(self, changed, values):
        """layerChanged: vertex changed[i] gets values[i]"""
        ch = np.asarray(changed, np.uint32)
        vals = np.broadcast_to(np.asarray(values, np.float32), ch.shape).copy()
        if ch.size:
            self.mm.layerChanged(ch, vals, self.factor)
            self.vc[ch] = vals

    def repair_and_check(self, seeds, rows, changed, oracle_rows=None):
        """repairs rows (a dict of dist / pred, in place) and checks them; returns the repair's stats and the fresh ones"""
        got = self.pl.dijkstraBatchRepair(seeds, changed, rows["dist"], rows["pred"])
        assert got["outcome"] == 0
        ref = self.fresh(seeds)
        for k in range(len(seeds)):
            assert _same(rows["dist"][k], ref["dist"][k]), f"row {k} (seed {seeds[k]}): dist"
            assert (rows["pred"][k] == ref["pred"][k]).all(), f"row {k} (seed {seeds[k]}): pred"
        if self.oracle:
            vc, w = self.mm.costs()
            for k in (range(len(seeds)) if oracle_rows is None else oracle_rows):
                o = self.om.dijkstra(w, vc, int(seeds[k]), invalid=self.invalid, cost_limit=self.cost_limit)
                assert _same(rows["dist"][k], np.asarray(o["dist"], np.float32)), f"row {k}: oracle dist"
                assert (rows["pred"][k] == o["pred"]).all(), f"row {k}: oracle pred"
        return got, ref

    def disc(self, centre, radius):
        d = np.linalg.norm(self.pos[:, :2] - np.asarray(centre, np.float32)[None, :2], axis=1)
        return np.where(d <= radius)[0].astype(np.uint32)

    def extent(self):
        return self.pos[:, :2].min(0), self.pos[:, :2].max(0)


def _base_costs(pos, rng):
    return (rng.random(pos.shape[0]) * 0.6).astype(np.float32)


MESHES = ["terrain", "planar", "exact_ties", "delaunay", "invalid"]


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
@pytest.mark.parametrize("mesh", MESHES)
def test_repair_disc_obstacle(api, oracle_mod, mesh, factor):
    """a disc obstacle appears (+inf, then just above the cost limit), disappears, moves: one update -> repair cycle
    after the other on the same rows"""
    rng = np.random.default_rng(1)
    pos, faces = _mesh("terrain" if mesh == "invalid" else mesh)
    invalid = (rng.random(pos.shape[0]) < 0.02).astype(np.uint8) if mesh == "invalid" else None
    costs = np.zeros(pos.shape[0], np.float32) if mesh == "exact_ties" else _base_costs(pos, rng)
    cost_limit = {"terrain": 1.0, "planar": 0.5, "exact_ties": 1.0, "delaunay": 0.45, "invalid": 1.0}[mesh]
    cs = Case(api, oracle_mod, pos, faces, costs, factor, invalid, cost_limit)
    lo, hi = cs.extent()
    at = lambda fx, fy: lo + (hi - lo) * np.array([fx, fy])
    seeds = np.array([centre_seed(pos, faces, f)[0] for f in ((0.3, 0.4), (0.7, 0.6), (0.5, 0.2))], np.uint32)
    rows = cs.fresh(seeds)
    disc = cs.disc(at(0.5, 0.5), 0.35)
    old = cs.vc[disc].copy()
    cs.update(disc, np.inf)                                          # appears
    cs.repair_and_check(seeds, rows, disc)
    cs.update(disc, np.float32(cost_limit) + np.float32(0.01))       # just above the cost limit: labelled, not expanded
    cs.repair_and_check(seeds, rows, disc)
    cs.update(disc, old)                                             # disappears: decreases only
    cs.repair_and_check(seeds, rows, disc)
    moved = cs.disc(at(0.55, 0.45), 0.35)                            # moves: the old disc clears, the new one blocks
    cs.update(moved, np.inf)
    cs.repair_and_check(seeds, rows, moved)
    back = np.setdiff1d(moved, cs.disc(at(0.6, 0.4), 0.35))
    nxt = cs.disc(at(0.6, 0.4), 0.35)
    cs.update(back, old[:1].repeat(back.size))
    cs.update(nxt, np.inf)
    cs.repair_and_check(seeds, rows, np.concatenate([back, nxt]))
    cs.mm.close()


def _corridor(api, oracle_mod, factor, closed):
    """a +inf wall across the map with one corridor, open or closed"""
    pos, faces = mesh_case(40, False)
    rng = np.random.default_rng(4)
    costs = _base_costs(pos, rng)
    x, y = pos[:, 0], pos[:, 1]
    wall = (x > 1.9) & (x < 2.15)
    gate = wall & (y > 1.6) & (y < 2.1)
    costs[wall & ~gate] = np.inf
    if closed:
        costs[gate] = np.inf
    cs = Case(api, oracle_mod, pos, faces, costs, factor)
    return cs, np.where(gate)[0].astype(np.uint32), costs


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
def test_repair_wall_and_gate(api, oracle_mod, factor):
    """a wall closes the corridor (the far side becomes unreachable: +inf and pred = self), then the gate opens again
    (unreached vertices become reachable)"""
    cs, gate, costs = _corridor(api, oracle_mod, factor, closed=False)
    seeds = np.array([centre_seed(cs.pos, cs.faces, (0.2, 0.5))[0], centre_seed(cs.pos, cs.faces, (0.8, 0.3))[0]], np.uint32)
    rows = cs.fresh(seeds)
    far = cs.pos[:, 0] > 2.3
    assert np.isfinite(rows["dist"][0][far]).any()
    cs.update(gate, np.inf)
    cs.repair_and_check(seeds, rows, gate)
    unreached = np.isinf(rows["dist"][0]) & far
    assert unreached.any() and (rows["pred"][0][unreached] == np.where(unreached)[0]).all()
    cs.update(gate, 0.1)
    cs.repair_and_check(seeds, rows, gate)
    assert np.isfinite(rows["dist"][0][far]).any()
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
def test_repair_change_kinds(api, oracle_mod, factor):
    """scattered single vertices; a change at a seed; every vertex changed; duplicates and unchanged vertices in the
    changed list; n_changed == 0 leaves the rows untouched"""
    rng = np.random.default_rng(7)
    pos, faces = mesh_case(32, True)
    cs = Case(api, oracle_mod, pos, faces, _base_costs(pos, rng), factor, cost_limit=0.5)
    V = cs.om.V
    seeds = rng.choice(V, 5, replace=False).astype(np.uint32)
    rows = cs.fresh(seeds)
    sc = rng.choice(V, 25, replace=False).astype(np.uint32)
    cs.update(sc, (rng.random(sc.size) * 0.9).astype(np.float32))
    cs.repair_and_check(seeds, rows, sc)
    cs.update(seeds[:2], [0.55, 0.2])                               # at a seed: over the limit (no expansion), then cheap
    cs.repair_and_check(seeds, rows, seeds[:2])
    allv = np.arange(V, dtype=np.uint32)
    cs.update(allv, _base_costs(pos, rng))
    cs.repair_and_check(seeds, rows, allv)
    ch = rng.choice(V, 12, replace=False).astype(np.uint32)
    cs.update(ch, 0.45)
    listed = np.concatenate([ch, ch[:5], rng.choice(V, 10, replace=False).astype(np.uint32), ch[::-1]])
    cs.repair_and_check(seeds, rows, listed)
    before = (rows["dist"].copy(), rows["pred"].copy())
    got = cs.pl.dijkstraBatchRepair(seeds, np.empty(0, np.uint32), rows["dist"], rows["pred"])
    assert got["outcome"] == 0 and _same(rows["dist"], before[0]) and (rows["pred"] == before[1]).all()
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
def test_repair_two_regions(api, oracle_mod, factor):
    """two changed regions at very different distances from the seed, one lowering and one raising costs: the far region
    must be reached although the band starts at the near one"""
    rng = np.random.default_rng(12)
    pos, faces = mesh_case(48, True)
    cs = Case(api, oracle_mod, pos, faces, _base_costs(pos, rng), factor)
    lo, hi = cs.extent()
    s = centre_seed(pos, faces, (0.1, 0.1))[0]
    seeds = np.array([s, centre_seed(pos, faces, (0.15, 0.12))[0]], np.uint32)
    rows = cs.fresh(seeds)
    near = cs.disc(lo + (hi - lo) * 0.15, 0.2)
    far = cs.disc(lo + (hi - lo) * 0.9, 0.3)
    for near_v, far_v in ((0.0, np.inf), (np.inf, 0.0), (0.9, 0.05)):
        cs.update(near, near_v); cs.update(far, far_v)
        cs.repair_and_check(seeds, rows, np.concatenate([near, far]))
    far_only = cs.disc(lo + (hi - lo) * 0.85, 0.2)                   # a single far region: the whole band is empty before it
    cs.update(far_only, 0.0)
    cs.repair_and_check(seeds, rows, far_only)
    cs.mm.close()


@pytest.mark.gpu
def test_repair_union_of_updates(api, oracle_mod):
    """one repair after three updates, with the union of their changed sets (overlapping, in any order)"""
    rng = np.random.default_rng(13)
    pos, faces = mesh_case(36, True)
    cs = Case(api, oracle_mod, pos, faces, _base_costs(pos, rng), 1.0)
    V = cs.om.V
    seeds = rng.choice(V, 6, replace=False).astype(np.uint32)
    rows = cs.fresh(seeds)
    sets = []
    for c, val in (((0.3, 0.3), np.inf), ((0.35, 0.3), 0.0), ((0.7, 0.6), 0.8)):
        lo, hi = cs.extent()
        d = cs.disc(lo + (hi - lo) * np.array(c), 0.3)
        cs.update(d, val)
        sets.append(d)
    union = np.concatenate(sets[::-1])
    rng.shuffle(union)
    cs.repair_and_check(seeds, rows, union)
    cs.mm.close()


@pytest.mark.gpu
def test_repair_inflation_chain(api, oracle_mod):
    """the library's own update set: InflationLayer.onInputChanged -> layerChanged(changed) -> repair, three cycles of
    moving lethal discs"""
    from tests.util import disc_lethals
    pos, faces = mesh_case(40, True)
    cs = Case(api, oracle_mod, pos, faces, np.zeros(pos.shape[0], np.float32), 1.0, cost_limit=0.95)
    infl = api.InflationLayer(cs.mm)
    rng = np.random.default_rng(3)
    seeds = rng.choice(cs.om.V, 4, replace=False).astype(np.uint32)
    rows = cs.fresh(seeds)
    for cyc in range(3):
        lethals = disc_lethals(pos, 4, 0.25, seed=100 + cyc)
        got = infl.onInputChanged(lethals)
        assert got["changed"].size > 0
        cs.mm.layerChanged(got["changed"], got["cost"], cs.factor, by_vertex=True, default_value=0.0)
        cs.repair_and_check(seeds, rows, got["changed"])
    cs.mm.close()


@pytest.mark.gpu
def test_repair_pointer_modes_and_sources(api, oracle_mod):
    """device rows repaired in place give the same bytes as host rows; duplicate seeds; rows that came from single
    full-field mnb_dijkstra calls are valid input"""
    rng = np.random.default_rng(8)
    pos, faces = mesh_case(30, True)
    cs = Case(api, oracle_mod, pos, faces, _base_costs(pos, rng), 1.0)
    V = cs.om.V
    seeds = np.array([5, 400, 5, 777, 400], np.uint32)
    rows = cs.fresh(seeds)
    single = dict(dist=np.stack([cs.pl.dijkstra(int(s))["dist"] for s in seeds]),
                  pred=np.stack([cs.pl.dijkstra(int(s))["pred"] for s in seeds]))
    assert _same(single["dist"], rows["dist"]) and (single["pred"] == rows["pred"]).all()
    host = dict(dist=rows["dist"].copy(), pred=rows["pred"].copy())
    d = cs.disc(cs.pos[400, :2], 0.3)
    cs.update(d, np.inf)
    cs.repair_and_check(seeds, host, d)
    cs.repair_and_check(seeds, single, d)
    on_gpu = not hasattr(cs.mm.L, "mnb_emu_switch")
    if on_gpu:
        import torch
        dd = torch.from_numpy(rows["dist"]).cuda(); dp = torch.from_numpy(rows["pred"].view(np.int32)).cuda()
        pd, pp = dd.data_ptr(), dp.data_ptr()
        back = lambda: (dd.cpu().numpy(), dp.cpu().numpy().view(np.uint32))
    else:
        dd, dp = rows["dist"].copy(), rows["pred"].copy()
        pd, pp = dd.ctypes.data, dp.ctypes.data
        back = lambda: (dd, dp)
    cs.mm.use_device_pointers(True)
    try:
        assert cs.mm.dijkstra_batch_repair_dev(seeds, d, cs.cost_limit, pd, pp) == 0
        if on_gpu:
            torch.cuda.synchronize()
    finally:
        cs.mm.use_device_pointers(False)
    gd, gp = back()
    assert _same(gd, host["dist"]) and (gp == host["pred"]).all()
    cs.mm.close()


@pytest.mark.gpu
def test_repair_keeps_state(api, oracle_mod):
    """a repair leaves the last mnb_cvp's back-tracking path and the last inflation's vector map alone"""
    rng = np.random.default_rng(21)
    pos, faces = mesh_case(40, True)
    costs = (0.45 + 0.45 * np.sin(3.0 * pos[:, 0])).astype(np.float32)
    cs = Case(api, oracle_mod, pos, faces, costs, 1.0)
    cpl = api.CVPMeshPlanner(cs.mm)
    infl = api.InflationLayer(cs.mm)
    sv, sf, sp = centre_seed(pos, faces, (0.2, 0.25))
    rv, rf, rp = centre_seed(pos, faces, (0.8, 0.7))
    seeds = rng.choice(cs.om.V, 4, replace=False).astype(np.uint32)
    rows = cs.fresh(seeds)
    ch = cs.disc(pos[seeds[0], :2], 0.3)
    cs.update(ch, np.inf)
    assert cpl.waveFrontPropagation(sf, sp, rf)["outcome"] == 0
    bt0 = cpl.backtrack(rp, rf)
    infl.waveCostInflation(np.array([sv, rv], np.uint32))
    iv0 = infl.vectorMap()
    cs.repair_and_check(seeds, rows, ch)
    bt1 = cpl.backtrack(rp, rf)
    assert bt0["outcome"] == bt1["outcome"] == 0 and len(bt0["positions"]) > 5
    assert _same(bt0["positions"], bt1["positions"]) and (bt0["faces"] == bt1["faces"]).all()
    assert _same(iv0, infl.vectorMap())
    cs.mm.close()


def _raw(mm, seeds, changed, dist, pred, cost_limit=1.0, seeds_ptr=True, changed_ptr=True):
    sv = np.ascontiguousarray(seeds, np.uint32); ch = np.ascontiguousarray(changed, np.uint32)
    p = lambda a, on=True: a.ctypes.data_as(C.c_void_p) if (on and a is not None) else None
    return mm.L.mnb_dijkstra_batch_repair(mm._ctx, sv.size, p(sv, seeds_ptr), float(cost_limit), ch.size, p(ch, changed_ptr),
                                          p(dist), p(pred))


@pytest.mark.gpu
def test_repair_arguments(api, oracle_mod):
    """no costs -> MNB_E_STATE (-3); n == 0, a NULL array or a changed vertex >= V -> MNB_E_ARG (-1); a seed >= V ->
    INVALID_START (52); nothing is written in any of these"""
    pos, faces = mesh_case(20, True)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    V = om.V
    dist = np.full((2, V), 7.0, np.float32); pred = np.full((2, V), 7, np.uint32)
    untouched = lambda: (dist == 7.0).all() and (pred == 7).all()
    assert _raw(mm, [3, 4], [5], dist, pred) == -3 and untouched()
    vc = np.zeros(V, np.float32)
    mm.setCosts(vc, om.edge_distances())
    assert _raw(mm, [3, 4], [5], None, pred) == -1 and untouched()
    assert _raw(mm, [3, 4], [5], dist, None) == -1 and untouched()
    assert _raw(mm, [3, 4], [5], dist, pred, seeds_ptr=False) == -1 and untouched()
    assert _raw(mm, [3, 4], [5], dist, pred, changed_ptr=False) == -1 and untouched()
    assert _raw(mm, [], [5], dist, pred) == -1 and untouched()
    assert _raw(mm, [3, 4], [5, V], dist, pred) == -1 and untouched()
    assert _raw(mm, [3, V], [5], dist, pred) == 52 and untouched()
    assert _raw(mm, [3, 4], [], dist, pred) == 0 and untouched()
    pl = api.DijkstraMeshPlanner(mm)
    rows = pl.dijkstraBatch([3, 4])
    d, p = rows["dist"].copy(), rows["pred"].copy()
    assert _raw(mm, [3, 4], [5, 6], d, p) == 0 and _same(d, rows["dist"]) and (p == rows["pred"]).all()
    with pytest.raises(ValueError):
        pl.dijkstraBatchRepair([3, 4], [5], d[:1], p)
    mm.close()


@pytest.mark.gpu
def test_repair_cancel(api, oracle_mod):
    """mnb_cancel from another thread -> CANCELED (51); the rows are then recomputed, and the next repair is exact"""
    pos, faces = mesh_case(120, True)
    cs = Case(api, oracle_mod, pos, faces, np.zeros(pos.shape[0], np.float32), 1.0, oracle=False)
    cs.mm.set_tuning(0.005, 1, 0)      # narrow band: many rounds per wave
    V = cs.om.V
    allv = np.arange(V, dtype=np.uint32)
    rng = np.random.default_rng(2)
    n = 8
    while True:                        # grow the batch until a repair of every vertex takes long enough to cancel
        seeds = rng.integers(0, V, n).astype(np.uint32)
        rows = cs.fresh(seeds)
        cs.pl.dijkstraBatchRepair(seeds, allv, rows["dist"], rows["pred"])       # warm at this size
        t0 = time.perf_counter(); full = cs.pl.dijkstraBatchRepair(seeds, allv, rows["dist"], rows["pred"])
        t_full = time.perf_counter() - t0
        assert full["outcome"] == 0
        if t_full > 0.2 or n >= 4096:
            break
        n *= 4
    assert t_full > 0.05, t_full
    outcomes = []

    def run():
        t1 = time.perf_counter(); o = cs.pl.dijkstraBatchRepair(seeds, allv, rows["dist"], rows["pred"])["outcome"]
        outcomes.append((o, time.perf_counter() - t1))
    t = threading.Thread(target=run)
    t.start(); time.sleep(0.25 * t_full); cs.mm.cancel(); t.join()
    assert outcomes[0][0] == 51, outcomes
    assert outcomes[0][1] < 0.85 * t_full, (outcomes, t_full)
    rows = cs.fresh(seeds[:3])
    sub = seeds[:3]
    d = cs.disc(cs.pos[sub[0], :2], 0.5)
    cs.update(d, np.inf)
    cs.repair_and_check(sub, rows, d)
    cs.mm.close()


@pytest.mark.gpu
def test_repair_work(api, oracle_mod):
    """a local change re-runs a small region: far fewer recomputes and settled vertices than the fresh batch"""
    rng = np.random.default_rng(9)
    pos, faces = mesh_case(90, True)
    cs = Case(api, oracle_mod, pos, faces, _base_costs(pos, rng), 1.0, oracle=False)
    seeds = rng.choice(cs.om.V, 6, replace=False).astype(np.uint32)
    rows = cs.fresh(seeds)
    lo, hi = cs.extent()
    d = cs.disc(lo + (hi - lo) * 0.92, 0.2)                          # near a corner: a small shadow behind it
    cs.update(d, np.inf)
    got, ref = cs.repair_and_check(seeds, rows, d)
    ratio = got["recomputes"] / ref["recomputes"]
    print(f"recomputes {got['recomputes']} of {ref['recomputes']} ({ratio:.3f}), settled {got['settled']} of "
          f"{ref['settled']}, rounds {got['rounds']} of {ref['rounds']}")
    assert ratio < 0.2 and got["settled"] < ref["settled"], ratio
    assert got["kernel_launches"] == 1
    cs.mm.close()


@pytest.mark.gpu
def test_repair_large_mesh(api, oracle_mod):
    """1 M-vertex terrain, 32 seeds: a disc obstacle appears, then moves; sampled rows against the oracle"""
    pos, faces = mesh_case(1000, True)
    cs = Case(api, oracle_mod, pos, faces, np.zeros(pos.shape[0], np.float32), 1.0)
    seeds = synth.batch_goal_vertices(cs.om.V, 32, seed=1234).astype(np.uint32)
    rows = cs.fresh(seeds)
    d1 = cs.disc(cs.pos[seeds[0], :2] + 2.0, 0.3)
    cs.update(d1, np.inf)
    cs.repair_and_check(seeds, rows, d1, oracle_rows=[0, 31])
    d2 = cs.disc(cs.pos[seeds[0], :2] + 2.3, 0.3)
    cs.update(d1, 0.0); cs.update(d2, np.inf)
    got, ref = cs.repair_and_check(seeds, rows, np.concatenate([d1, d2]), oracle_rows=[0])
    assert got["recomputes"] < ref["recomputes"]
    cs.mm.close()


def test_dijkstra_repair_on_the_cpu_interpreter():
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
