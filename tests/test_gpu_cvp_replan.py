"""CVP replanning (mnb_cvp_replan / CVPMeshPlanner.waveFrontReplan): a plan, mnb_update_vertex_costs calls, the replan --
then all four outputs and the return code bit for bit against a fresh mnb_cvp with the same arguments on the same context
and costs.  The GPU tests run with -m gpu on an H100; the CPU legs check the premise of the resume on the oracle and
replay the GPU tests on the CPU interpreter of the kernels (tests/emu)."""
import ctypes as C
import mmap
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
OUTS = ("dist", "pred", "direction", "cutting_face")
FIXTURES = ["deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour"]


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def _mesh(kind):
    if kind == "terrain":
        return mesh_case(32, True)
    if kind == "planar":
        return mesh_case(32, False)
    if kind == "exact_ties":
        return synth.grid_mesh(30, 30, jitter=0.0, terrain=False)
    if kind == "delaunay":
        return delaunay_mesh(900, seed=5, extent=3.2)
    raise ValueError(kind)


class Case:
    """one map and planner; `pending` collects the changed vertices since the last replan"""

    def __init__(self, api, oracle_mod, pos, faces, costs=None, factor=1.0, invalid=None, cost_limit=1.0, weights=None,
                 goal_dist_offset=0.3):
        self.api, self.pos, self.faces, self.factor = api, pos, faces, factor
        self.om = oracle_mod.OracleMesh(pos, faces)
        self.mm = api.MeshMap(pos, faces)
        self.V = self.om.V
        self.vc = np.zeros(self.V, np.float32) if costs is None else np.asarray(costs, np.float32).copy()
        self.ed = self.om.edge_distances()
        w = self.om.edge_weights(self.vc, self.ed, factor) if weights is None else weights
        self.invalid = invalid
        self.mm.setCosts(self.vc, w, invalid)
        self.pl = api.CVPMeshPlanner(self.mm, cost_limit=cost_limit, goal_dist_offset=goal_dist_offset)
        self.pending = []

    def update(self, changed, values):
        ch = np.asarray(changed, np.uint32)
        vals = np.broadcast_to(np.asarray(values, np.float32), ch.shape).copy()
        if ch.size:
            self.mm.layerChanged(ch, vals, self.factor)
            self.vc[ch] = vals
            self.pending.append(ch)

    def replan(self, sf, sp, rf=-1, extra=()):
        """the replan with the pending changes (plus `extra`) against a fresh mnb_cvp; returns both results"""
        ch = np.concatenate(self.pending + [np.asarray(extra, np.uint32)]) if self.pending or len(extra) else np.empty(0, np.uint32)
        got = self.pl.waveFrontReplan(sf, sp, rf, ch)
        self.pending = []
        ref = self.pl.waveFrontPropagation(sf, sp, rf)
        assert got["outcome"] == ref["outcome"], (got["outcome"], ref["outcome"])
        for k in OUTS:
            assert _same(got[k], ref[k]), f"{k}: {np.count_nonzero(got[k].view(np.uint32) != ref[k].view(np.uint32))} differ"
        return got, ref

    def disc(self, centre, radius):
        d = np.linalg.norm(self.pos[:, :2] - np.asarray(centre, np.float32)[None, :2], axis=1)
        return np.where(d <= radius)[0].astype(np.uint32)

    def at(self, fx, fy):
        lo, hi = self.pos[:, :2].min(0), self.pos[:, :2].max(0)
        return lo + (hi - lo) * np.array([fx, fy], np.float32)

    def face_at(self, fx, fy):
        return centre_seed(self.pos, self.faces, (fx, fy))


@pytest.mark.gpu
def test_replan_first_call_and_fallbacks(api, oracle_mod):
    """no resident wave, mnb_set_costs / mnb_compute_edge_weights in between, another seed, another cost limit: one whole
    wave each (settled == the fresh plan's); a matching call resumes"""
    rng = np.random.default_rng(3)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    _, sf, sp = cs.face_at(0.3, 0.3)
    _, sf2, sp2 = cs.face_at(0.6, 0.4)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.update(cs.disc(cs.at(0.8, 0.8), 0.2), 0.7)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] < ref["settled"]
    cs.mm.setCosts(cs.vc, cs.om.edge_weights(cs.vc, cs.ed, cs.factor))
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.mm.computeEdgeWeights(cs.vc, cs.factor)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    got, ref = cs.replan(sf2, sp2)                                   # another seed
    assert got["settled"] == ref["settled"]
    got, ref = cs.replan(sf2, sp2 + np.float32(1e-3))                # another seed position
    assert got["settled"] == ref["settled"]
    got, ref = cs.replan(sf2, sp2 + np.float32(1e-3))                # the same call again: nothing to re-run
    assert got["settled"] == 0
    cs.pl.cost_limit = 0.45                                          # another cost limit
    got, ref = cs.replan(sf2, sp2 + np.float32(1e-3))
    assert got["settled"] == ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("robot", [False, True])
@pytest.mark.parametrize("factor", [0.0, 1.0])
@pytest.mark.parametrize("mesh", ["terrain", "planar", "exact_ties", "delaunay", "invalid"])
def test_replan_changes(api, oracle_mod, mesh, factor, robot):
    """a chain of twelve updates and replans: changes near the robot, in mid-field, touching the seed face's ring,
    beyond the old cutoff; rises, drops, values crossing the cost limit and +inf; a new robot face beyond the old cutoff"""
    rng = np.random.default_rng(11)
    pos, faces = _mesh("terrain" if mesh == "invalid" else mesh)
    invalid = (rng.random(pos.shape[0]) < 0.02).astype(np.uint8) if mesh == "invalid" else None
    costs = np.zeros(pos.shape[0], np.float32) if mesh == "exact_ties" else (rng.random(pos.shape[0]) * 0.6).astype(np.float32)
    cs = Case(api, oracle_mod, pos, faces, costs, factor, invalid, cost_limit=0.9)
    sv, sf, sp = cs.face_at(0.2, 0.25)
    if invalid is not None:
        invalid[faces[sf]] = 0
        cs.mm.setCosts(cs.vc, cs.om.edge_weights(cs.vc, cs.ed, factor), invalid)
    rf = cs.face_at(0.65, 0.6)[1] if robot else -1
    rf_far = cs.face_at(0.9, 0.85)[1] if robot else -1
    cs.replan(sf, sp, rf)
    robot_xy = cs.at(0.65, 0.6)
    steps = [
        (cs.disc(robot_xy + 0.25, 0.12), np.inf),                    # near the robot
        (cs.disc(robot_xy + 0.25, 0.12), 0.0),                       # and gone again
        (cs.disc(cs.at(0.45, 0.45), 0.15), 0.95),                    # mid-field, over the cost limit
        (cs.disc(cs.at(0.45, 0.45), 0.15), 0.3),                     # back under it
        (cs.disc(cs.at(0.5, 0.3), 0.2), 0.05),                       # a drop
        (np.asarray(faces[sf], np.uint32), 0.2),                     # the seed face's ring
        (cs.disc(cs.at(0.92, 0.9), 0.15), 0.8),                      # beyond the old cutoff
        (rng.choice(cs.V, 25, replace=False).astype(np.uint32), 0.5),
        (cs.disc(robot_xy - 0.2, 0.1), 0.89999),                     # just under the limit
        (cs.disc(robot_xy - 0.2, 0.1), 0.9),                         # at it
        (cs.disc(cs.at(0.3, 0.7), 0.25), np.inf),
        (cs.disc(cs.at(0.3, 0.7), 0.25), 0.1),
    ]
    resumed = 0
    for i, (ch, val) in enumerate(steps):
        cs.update(ch, val)
        got, ref = cs.replan(sf, sp, rf_far if (robot and i == 7) else rf)
        resumed += got["settled"] < ref["settled"]
    got, ref = cs.replan(sf, sp, rf)                                 # only the robot face changed back
    assert resumed >= 4, resumed
    cs.mm.close()


def _fixture(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", f"fuzz_{name}.npz"))
    inv = d["inv"] if d["inv"].size else None
    return d["pos"], d["faces"], d["vc"], d["w"], inv, int(d["sf"]), d["sp"], int(d["rf"]), float(d["cl"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_replan_fixtures(api, oracle_mod, name):
    """the fuzz fixtures with deep cascades, a cascade-armed cutoff and a seed that pops after its neighbour: changes at
    the vertices right after the deepest back-steps, then at several depths of the pop order, with and without the cutoff"""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fixture(name)
    cs = Case(api, oracle_mod, pos, faces, vc, 1.0, inv, cost_limit=cl, weights=w)
    for robot in ([rf, -1] if rf >= 0 else [-1]):
        base, _ = cs.replan(sf, sp, robot)
        d = base["dist"]
        fin = np.where(np.isfinite(d))[0]
        order = fin[np.argsort(d[fin], kind="stable")]
        # a back-step: a vertex whose potential is below its predecessor's; change the vertices popped right after it
        back = fin[d[fin] < d[base["pred"][fin]]]
        picks = [order[np.searchsorted(d[order], d[v], side="right"):][:3] for v in back[:4]]
        picks += [order[int(q * (order.size - 1)):][:4] for q in (0.1, 0.5, 0.9)]
        for k, ch in enumerate(picks):
            cs.update(ch, (vc[ch] + 0.05 * (k + 1)) % cl)
            cs.replan(sf, sp, robot)
    cs.mm.close()


@pytest.mark.gpu
def test_replan_between_other_calls(api, oracle_mod):
    """mnb_cvp, the batch calls, the matrices, Dijkstra (single, batch and repair), inflation and inflation repair between
    two replans: the resident wave still resumes, and the result is exact"""
    rng = np.random.default_rng(5)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    sv, sf, sp = cs.face_at(0.3, 0.3)
    rv, rf, rp = cs.face_at(0.7, 0.7)
    cs.replan(sf, sp, rf)
    dij = api.DijkstraMeshPlanner(cs.mm)
    infl = api.InflationLayer(cs.mm)
    others = [
        lambda: cs.pl.waveFrontPropagation(rf, rp),
        lambda: cs.pl.waveFrontPropagationBatch([sf, rf], np.stack([sp, rp])),
        lambda: cs.pl.waveFrontPropagationBatchFields([sf, rf], np.stack([sp, rp])),
        lambda: cs.pl.costMatrix([sf, rf], np.stack([sp, rp]), [sv, rv]) if hasattr(cs.pl, "costMatrix") else None,
        lambda: dij.dijkstra(int(rv)),
        lambda: dij.costMatrix([sv, rv], [rv, sv]),
        lambda: dij.dijkstraBatchRepair([sv], [rv], *[dij.dijkstraBatch([sv])[k] for k in ("dist", "pred")]),
        lambda: infl.waveCostInflation(np.array([rv], np.uint32)),
        lambda: infl.repairInflation(np.array([rv, sv], np.uint32)),
    ]
    for k, other in enumerate(others):
        cs.update(cs.disc(cs.at(0.6, 0.62), 0.08 + 0.01 * k), 0.3 + 0.05 * k)
        other()
        got, ref = cs.replan(sf, sp, rf)
        assert got["settled"] < ref["settled"], k
    cs.mm.close()


@pytest.mark.gpu
def test_replan_pointer_modes(api, oracle_mod):
    """device-pointer outputs (NULL outputs included) equal the host-pointer replan of a second context with the same history"""
    rng = np.random.default_rng(8)
    pos, faces = _mesh("terrain")
    costs = (rng.random(pos.shape[0]) * 0.5).astype(np.float32)
    a = Case(api, oracle_mod, pos, faces, costs)
    b = Case(api, oracle_mod, pos, faces, costs)
    _, sf, sp = a.face_at(0.25, 0.3)
    rf = a.face_at(0.7, 0.75)[1]
    on_gpu = not hasattr(b.mm.L, "mnb_emu_switch")
    for step in range(3):
        ch = a.disc(a.at(0.5 + 0.05 * step, 0.5), 0.12)
        a.update(ch, 0.6); b.update(ch, 0.6)
        got, _ = a.replan(sf, sp, rf)
        pend = np.concatenate(b.pending); b.pending = []
        if on_gpu:
            import torch
            bufs = [torch.empty(b.V, dtype=t, device="cuda") for t in (torch.float32, torch.int32, torch.float32, torch.int32)]
            ptrs = [x.data_ptr() for x in bufs]
            back = lambda: [bufs[0].cpu().numpy(), bufs[1].cpu().numpy().view(np.uint32), bufs[2].cpu().numpy(), bufs[3].cpu().numpy()]
        else:
            # the interpreter runs a cooperative or cluster launch as one forked process per CTA: what such a kernel
            # writes reaches the caller's memory only when that memory is shared
            bufs = [np.frombuffer(mmap.mmap(-1, 4 * b.V), t, b.V) for t in (np.float32, np.uint32, np.float32, np.int32)]
            ptrs = [x.ctypes.data for x in bufs]
            back = lambda: bufs
        if step == 2:
            ptrs[2] = 0                                               # a NULL output
        b.mm.use_device_pointers(True)
        try:
            rc = b.mm.cvp_replan_dev(sf, sp, rf, b.pl.cost_limit, b.pl.goal_dist_offset, pend, *ptrs)
            if on_gpu:
                torch.cuda.synchronize()
        finally:
            b.mm.use_device_pointers(False)
        assert rc == got["outcome"]
        for k, x in zip(OUTS, back()):
            if not (step == 2 and k == "direction"):
                assert _same(x, got[k]), k
    a.mm.close(); b.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [-1, 1, 2, 4, 8, 16])
def test_replan_launch_forms(api, oracle_mod, cluster):
    """the whole-grid kernel and every cluster size of the single-plan kernel resume exactly"""
    rng = np.random.default_rng(12)
    pos, faces = _mesh("delaunay")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.6).astype(np.float32))
    cs.mm.set_tuning(0.0 if cluster == -1 else 0.3, cluster, 0)
    _, sf, sp = cs.face_at(0.2, 0.3)
    rf = cs.face_at(0.75, 0.7)[1]
    for robot in (-1, rf):
        cs.replan(sf, sp, robot)
        for k in range(3):
            cs.update(cs.disc(cs.at(0.4 + 0.15 * k, 0.5), 0.2), [np.inf, 0.2, 0.05][k])
            got, ref = cs.replan(sf, sp, robot)
    assert got["settled"] < ref["settled"]
    cs.mm.close()


def _raw(mm, sf, sp, rf, changed, outs, changed_ptr=True, cost_limit=1.0):
    ch = np.ascontiguousarray(changed, np.uint32); sp = np.ascontiguousarray(sp, np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    return mm.L.mnb_cvp_replan(mm._ctx, int(sf), p(sp), int(rf), float(cost_limit), 0.3, ch.size, p(ch) if changed_ptr else None,
                               *[p(o) for o in outs])


@pytest.mark.gpu
def test_replan_arguments(api, oracle_mod):
    """no costs -> MNB_E_STATE (-3); a changed vertex >= V or a NULL changed list with n > 0 -> MNB_E_ARG (-1); a seed
    or robot face >= F -> INVALID_START (52) / INVALID_GOAL (53); nothing is written in any of these"""
    pos, faces = mesh_case(16, True)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    V, F = om.V, faces.shape[0]
    outs = [np.full(V, 7, t) for t in (np.float32, np.uint32, np.float32, np.int32)]
    untouched = lambda: all((o == 7).all() for o in outs)
    sp = pos[faces[5]].mean(0)
    assert _raw(mm, 5, sp, -1, [1], outs) == -3 and untouched()
    mm.setCosts(np.zeros(V, np.float32), om.edge_distances())
    assert _raw(mm, 5, sp, -1, [1, V], outs) == -1 and untouched()
    assert _raw(mm, 5, sp, -1, [1], outs, changed_ptr=False) == -1 and untouched()
    assert _raw(mm, F, sp, -1, [1], outs) == 52 and untouched()
    assert _raw(mm, 5, sp, F, [1], outs) == 53 and untouched()
    assert _raw(mm, 5, sp, -1, [], outs) == 0 and not untouched()
    ref = api.CVPMeshPlanner(mm).waveFrontPropagation(5, sp)
    for k, o in zip(OUTS, outs):
        assert _same(o, ref[k]), k
    assert _raw(mm, 5, sp, -1, [], [None] * 4) == 0
    mm.close()


@pytest.mark.gpu
def test_replan_backtrack(api, oracle_mod):
    """replan + backtrack is makePlan: the path equals the one after a fresh mnb_cvp"""
    rng = np.random.default_rng(4)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.4).astype(np.float32))
    _, sf, sp = cs.face_at(0.2, 0.2)
    _, rf, rp = cs.face_at(0.8, 0.75)
    cs.replan(sf, sp, rf)
    for k in range(3):
        cs.update(cs.disc(cs.at(0.55 + 0.1 * k, 0.5), 0.15), np.inf)
        got = cs.pl.waveFrontReplan(sf, sp, rf, np.concatenate(cs.pending)); cs.pending = []
        assert got["outcome"] == 0
        bt = cs.pl.backtrack(rp, rf)
        assert cs.pl.waveFrontPropagation(sf, sp, rf)["outcome"] == 0
        ref = cs.pl.backtrack(rp, rf)
        assert bt["outcome"] == ref["outcome"] == 0 and len(bt["positions"]) > 5
        assert _same(bt["positions"], ref["positions"]) and (bt["faces"] == ref["faces"]).all()
    cs.mm.close()


@pytest.mark.gpu
def test_replan_resumes_large(api, oracle_mod):
    """250 k-vertex terrain, goal in the middle, with and without the robot cutoff: a change near the robot re-settles a
    small share of a fresh plan's vertices; a change touching the seed face's ring runs the whole wave"""
    pos, faces = mesh_case(500, True)
    cs = Case(api, oracle_mod, pos, faces)
    _, sf, sp = cs.face_at(0.5, 0.5)
    _, rf, rp = cs.face_at(0.85, 0.8)
    for robot in (rf, -1):
        cs.replan(sf, sp, robot)
        cs.update(cs.disc(cs.at(0.85, 0.8) + 1.5, 0.4), 0.8)
        got, ref = cs.replan(sf, sp, robot)
        print(f"robot {robot}: settled {got['settled']} of {ref['settled']}, rounds {got['rounds']} of {ref['rounds']}")
        assert got["settled"] < 0.5 * ref["settled"]
        cs.update(np.asarray(faces[sf], np.uint32), 0.1)
        got, ref = cs.replan(sf, sp, robot)
        if robot == -1:         # (with a cutoff, vertices settled before it is known settle again: the count varies)
            assert got["settled"] == ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
def test_replan_cancel(api, oracle_mod):
    """mnb_cancel from another thread -> CANCELED (51); the resident wave is dropped: the next call runs a whole wave"""
    pos, faces = mesh_case(400, True)
    cs = Case(api, oracle_mod, pos, faces)
    cs.mm.set_tuning(0.002, 1, 0)                                    # narrow band on one CTA: a slow wave
    _, sf, sp = cs.face_at(0.5, 0.5)
    allv = np.arange(cs.V, dtype=np.uint32)                          # T0 before the seeds: a whole wave in the resident workspace
    cs.replan(sf, sp)
    t0 = time.perf_counter(); whole = cs.pl.waveFrontReplan(sf, sp, -1, allv); t_full = time.perf_counter() - t0
    assert whole["outcome"] == 0 and t_full > 0.05, t_full
    outcomes = []
    t = threading.Thread(target=lambda: outcomes.append(cs.pl.waveFrontReplan(sf, sp, -1, allv)["outcome"]))
    t.start(); time.sleep(0.3 * t_full); cs.mm.cancel(); t.join()
    assert outcomes == [51]
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [-1, 1, 4])
def test_replan_pool_overflow_retry(api, oracle_mod, cluster):
    """a resumed wave that runs out of level pool (a test hook caps what it may add) is run again as one whole wave from an
    empty pool, in every launch form: the rows are exact, and the whole wave's settled count is the fresh plan's"""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fixture("deep_cascade_planar")
    cs = Case(api, oracle_mod, pos, faces, vc, 1.0, inv, cost_limit=cl, weights=w)
    cs.mm.set_tuning(0.0 if cluster == -1 else 0.3, cluster, 0)
    hook = cs.mm.L.mnb_debug_set_replan_pool_room
    hook.argtypes = [C.c_void_p, C.c_uint32]
    base, ref = cs.replan(sf, sp)
    assert ref["deep_labels"] > 0                                  # the wave has labels that live in the pool
    d = base["dist"]
    fin = np.where(np.isfinite(d))[0]
    order = fin[np.argsort(d[fin], kind="stable")]
    ch = order[int(0.1 * order.size):][:3]                          # early: the re-run tail holds nearly every deep label
    assert hook(cs.mm._ctx, 1) == 0
    try:
        cs.update(ch, (vc[ch] + 0.1) % cl)
        got, ref = cs.replan(sf, sp)
        assert got["settled"] == ref["settled"]                     # the whole wave ran (a resume settles fewer)
    finally:
        hook(cs.mm._ctx, 0)
    cs.update(ch, vc[ch])
    got, ref = cs.replan(sf, sp)                                    # the retried wave is resident: the next call resumes
    assert got["settled"] < ref["settled"]
    cs.mm.close()


def _pop_order(oracle_mod, om, w, vc, sf, sp, rf, off, inv, cl):
    """the oracle's plan and the sequence number of every vertex's pop (int64; never popped: 2^32 - 1)"""
    from oracle import oracle as O
    pop = np.full(om.V, 0xffffffff, np.uint32)
    O._lib.orc_debug_set_pop_buffer(pop.ctypes.data_as(C.c_void_p))
    try:
        r = om.cvp(w, vc, sf, sp, rf, invalid=inv, cost_limit=cl, goal_dist_offset=off)
    finally:
        O._lib.orc_debug_set_pop_buffer(None)
    return r, pop.astype(np.int64)


def _premise(oracle_mod, pos, faces, vc, factor, inv, sf, sp, cl, changed, new_vals, old_robot=(-1, 0.3), new_robot=(-1, 0.3)):
    """a fresh oracle run on the new costs with the new robot face and goal_dist_offset pops the same vertices in the same
    order, with the same four outputs, as the run on the old costs with the old ones, up to T0 = the earliest of: the first
    old pop in the closed 1-rings of the changed set, the old run's cutoff arming (the pop of the last robot vertex), and
    the new robot face's last pop in the old run.  Returns the size of that prefix."""
    om = oracle_mod.OracleMesh(pos, faces)
    ed = om.edge_distances()
    old, pop_old = _pop_order(oracle_mod, om, om.edge_weights(vc, ed, factor), vc, sf, sp, *old_robot, inv, cl)
    vc2 = vc.copy(); vc2[changed] = new_vals
    new, pop_new = _pop_order(oracle_mod, om, om.edge_weights(vc2, ed, factor), vc2, sf, sp, *new_robot, inv, cl)
    never = np.int64(0xffffffff)
    ring = set(int(c) for c in changed)
    for f in faces:
        if ring.intersection(int(x) for x in f):
            ring.update(int(x) for x in f)
    t0 = min([int(pop_old[v]) for v in ring] + [never])
    for rf, _ in (old_robot, new_robot):
        if rf >= 0:
            t0 = min(t0, int(pop_old[faces[rf]].max()))         # (never popped: 2^32 - 1, no bound)
    prefix = np.where(pop_old < t0)[0]
    assert (pop_new[prefix] == pop_old[prefix]).all()
    for k in OUTS:
        assert _same(old[k][prefix], new[k][prefix]), k
    return prefix.size


def test_oracle_replan_premise(oracle_mod):
    """the premise of the resume on the oracle (CPU): random changes on random maps and on the fuzz fixtures"""
    rng = np.random.default_rng(17)
    kept = 0
    for trial in range(12):
        pos, faces = mesh_case(26, bool(trial % 2), seed=trial)
        V = pos.shape[0]
        vc = (rng.random(V) * 0.6).astype(np.float32)
        inv = (rng.random(V) < 0.03).astype(np.uint8) if trial % 3 == 0 else None
        _, sf, sp = centre_seed(pos, faces, tuple(rng.random(2) * 0.6 + 0.2))
        if inv is not None:
            inv[faces[sf]] = 0
        ch = rng.choice(V, int(rng.integers(1, 30)), replace=False).astype(np.uint32)
        vals = rng.choice(np.array([0.0, 0.3, 0.95, np.inf], np.float32), ch.size)
        kept += _premise(oracle_mod, pos, faces, vc, float(trial % 2), inv, sf, sp, 0.9, ch, vals)
    for name in FIXTURES:
        pos, faces, vc, _, inv, sf, sp, rf, cl = _fixture(name)
        for q in (0.3, 0.7):
            v = int(np.argsort(np.linalg.norm(pos[:, :2] - pos[faces[sf]].mean(0)[:2], axis=1))[int(q * pos.shape[0])])
            kept += _premise(oracle_mod, pos, faces, vc, 1.0, inv, sf, sp, cl, np.array([v], np.uint32),
                             np.array([(vc[v] + 0.4) % cl], np.float32))
    assert kept > 0


def test_oracle_replan_premise_cutoff(oracle_mod):
    """the two cutoff terms of T0 on the oracle (CPU): the robot face and goal_dist_offset differ between the old and the
    new run -- a robot nearer to the goal, one farther away, a smaller and a larger offset, with and without a cost change,
    and the cascade-armed cutoff fixture"""
    rng = np.random.default_rng(23)
    kept = 0
    for trial in range(8):
        pos, faces = mesh_case(26, bool(trial % 2), seed=40 + trial)
        V = pos.shape[0]
        vc = (rng.random(V) * 0.6).astype(np.float32)
        _, sf, sp = centre_seed(pos, faces, (0.5, 0.5))
        rfs = [centre_seed(pos, faces, fr)[1] for fr in ((0.7, 0.65), (0.9, 0.85), (0.3, 0.6))]
        old_rf, new_rf = rfs[trial % 3], rfs[(trial + 1) % 3]
        offs = (0.3, [0.05, 0.3, 1.5][trial % 3])
        ch = rng.choice(V, 12, replace=False).astype(np.uint32) if trial % 2 else np.empty(0, np.uint32)
        vals = rng.choice(np.array([0.0, 0.95, np.inf], np.float32), ch.size)
        kept += _premise(oracle_mod, pos, faces, vc, 1.0, None, sf, sp, 0.9, ch, vals, (old_rf, offs[0]), (new_rf, offs[1]))
        kept += _premise(oracle_mod, pos, faces, vc, 1.0, None, sf, sp, 0.9, ch, vals, (-1, 0.3), (old_rf, offs[1]))
        kept += _premise(oracle_mod, pos, faces, vc, 1.0, None, sf, sp, 0.9, ch, vals, (old_rf, offs[0]), (-1, 0.3))
    pos, faces, vc, _, inv, sf, sp, rf, cl = _fixture("cutoff_cascade")
    other = centre_seed(pos, faces, (0.2, 0.8))[1]
    for new_robot in ((rf, 0.05), (other, 0.3), (-1, 0.3)):
        kept += _premise(oracle_mod, pos, faces, vc, 1.0, inv, sf, sp, cl, np.empty(0, np.uint32), np.empty(0, np.float32),
                         (rf, 0.3), new_robot)
    assert kept > 0


@pytest.mark.parametrize("shuffle, expr", [
    (None, "not large and not cancel"),
    ("5", "first_call or fixtures or launch_forms or overflow or backtrack or (changes and terrain)"),
])
def test_cvp_replan_on_the_cpu_interpreter(shuffle, expr):
    """the GPU tests above (minus the 250 k-vertex and the cancel test) with the kernels compiled by g++ against tests/emu,
    on 4 emulated SMs, in the default warp order; a third of them again in a randomised one.  One order per test, so each
    replay has the whole per-test time budget of the suite."""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    env = dict(os.environ, MNB_EMU_SMS="4", **({"MNB_EMU_SHUFFLE": shuffle} if shuffle else {}))
    r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider", "-k", expr],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=560)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"shuffle {shuffle}:\n{tail}"
