"""Batched CVP replanning (mnb_cvp_batch_replan / CVPMeshPlanner.waveFrontReplanBatch): a batch of goals, cost updates,
the batch replan -- then every requested row and the return code bit for bit against a fresh mnb_cvp_batch_fields with
the same goals on the same context and costs, run right after it.  The GPU tests run with -m gpu on an H100; the CPU leg
replays them on the CPU interpreter of the kernels (tests/emu)."""
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
FIXTURES = ["deep_cascade_planar", "deep_cascade_delaunay", "deep_cascade_maze", "seed_after_neighbour"]


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


def _fixture(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", f"fuzz_{name}.npz"))
    inv = d["inv"] if d["inv"].size else None
    return d["pos"], d["faces"], d["vc"], d["w"], inv, int(d["sf"]), d["sp"], float(d["cl"])


class Case:
    """one map and planner; `pending` collects the changed vertices since the last batch replan"""

    def __init__(self, api, oracle_mod, pos, faces, costs=None, factor=1.0, invalid=None, cost_limit=1.0, weights=None):
        self.api, self.pos, self.faces, self.factor = api, pos, faces, factor
        self.om = oracle_mod.OracleMesh(pos, faces)
        self.mm = api.MeshMap(pos, faces)
        self.V = self.om.V
        self.vc = np.zeros(self.V, np.float32) if costs is None else np.asarray(costs, np.float32).copy()
        self.ed = self.om.edge_distances()
        w = self.om.edge_weights(self.vc, self.ed, factor) if weights is None else weights
        self.mm.setCosts(self.vc, w, invalid)
        self.pl = api.CVPMeshPlanner(self.mm, cost_limit=cost_limit)
        self.pending = []

    def update(self, changed, values):
        ch = np.asarray(changed, np.uint32)
        vals = np.broadcast_to(np.asarray(values, np.float32), ch.shape).copy()
        if ch.size:
            self.mm.layerChanged(ch, vals, self.factor)
            self.vc[ch] = vals
            self.pending.append(ch)

    def replan(self, sf, sp, want=OUTS):
        """the batch replan with the pending changes against a fresh batch; returns both results"""
        ch = np.concatenate(self.pending) if self.pending else np.empty(0, np.uint32)
        got = self.pl.waveFrontReplanBatch(sf, sp, ch, want=want)
        self.pending = []
        ref = self.pl.waveFrontPropagationBatchFields(sf, sp, want=want)
        assert got["outcome"] == ref["outcome"], (got["outcome"], ref["outcome"])
        for k in want:
            assert _same(got[k], ref[k]), f"{k}: {np.count_nonzero(got[k].view(np.uint32) != ref[k].view(np.uint32))} differ"
        return got, ref

    def settled(self, sf, sp):
        """the settled count of a fresh batch of these goals"""
        return self.pl.waveFrontPropagationBatchFields(sf, sp, want=("dist",))["settled"]

    def disc(self, centre, radius):
        d = np.linalg.norm(self.pos[:, :2] - np.asarray(centre, np.float32)[None, :2], axis=1)
        return np.where(d <= radius)[0].astype(np.uint32)

    def at(self, fx, fy):
        lo, hi = self.pos[:, :2].min(0), self.pos[:, :2].max(0)
        return lo + (hi - lo) * np.array([fx, fy], np.float32)

    def goals(self, fracs):
        """seed faces and positions at the fractions (fx, fy) of the map"""
        got = [centre_seed(self.pos, self.faces, f) for f in fracs]
        return np.array([g[1] for g in got], np.uint32), np.stack([g[2] for g in got]).astype(np.float32)


def _spread(k, rng):
    return [tuple(x) for x in rng.random((k, 2)) * 0.8 + 0.1]


@pytest.mark.gpu
def test_batch_replan_first_call_and_fallbacks(api, oracle_mod):
    """no resident waves, mnb_set_costs / mnb_compute_edge_weights in between, another cost limit: whole waves (settled
    == the fresh batch's); a matching call after an update resumes; the same call again re-runs nothing; a moved seed
    position runs that goal alone whole"""
    rng = np.random.default_rng(3)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    sf, sp = cs.goals(_spread(8, rng))
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.update(cs.disc(cs.at(0.8, 0.8), 0.15), 0.7)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] < ref["settled"]
    got, ref = cs.replan(sf, sp)                                     # no change: nothing to re-run
    assert got["settled"] == 0
    cs.mm.setCosts(cs.vc, cs.om.edge_weights(cs.vc, cs.ed, cs.factor))
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.mm.computeEdgeWeights(cs.vc, cs.factor)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.pl.cost_limit = 0.45                                          # another cost limit
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    sp2 = sp.copy(); sp2[3] += np.float32(1e-3)                      # one goal's seed position moves
    got, ref = cs.replan(sf, sp2)
    assert got["settled"] == cs.settled(sf[3:4], sp2[3:4])
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
@pytest.mark.parametrize("mesh", ["terrain", "planar", "exact_ties", "delaunay", "invalid"])
def test_batch_replan_changes(api, oracle_mod, mesh, factor):
    """a chain of ten updates and batch replans with twelve goals spread over the map: changes on a seed face, near some
    goals and far from others; rises, drops, values crossing the cost limit, +inf walls that appear and disappear"""
    rng = np.random.default_rng(11)
    pos, faces = _mesh("terrain" if mesh == "invalid" else mesh)
    invalid = (rng.random(pos.shape[0]) < 0.02).astype(np.uint8) if mesh == "invalid" else None
    costs = np.zeros(pos.shape[0], np.float32) if mesh == "exact_ties" else (rng.random(pos.shape[0]) * 0.6).astype(np.float32)
    cs = Case(api, oracle_mod, pos, faces, costs, factor, invalid, cost_limit=0.9)
    sf, sp = cs.goals(_spread(12, rng))
    if invalid is not None:
        invalid[faces[sf].reshape(-1)] = 0
        cs.mm.setCosts(cs.vc, cs.om.edge_weights(cs.vc, cs.ed, factor), invalid)
    cs.replan(sf, sp)
    steps = [
        (cs.disc(cs.at(0.5, 0.5), 0.12), np.inf),                    # a wall
        (cs.disc(cs.at(0.5, 0.5), 0.12), 0.0),                       # and gone again
        (cs.disc(cs.at(0.3, 0.7), 0.15), 0.95),                      # over the cost limit
        (cs.disc(cs.at(0.3, 0.7), 0.15), 0.3),                       # back under it
        (cs.disc(cs.at(0.7, 0.3), 0.2), 0.05),                       # a drop
        (np.asarray(faces[sf[0]], np.uint32), 0.2),                  # a seed face
        (rng.choice(cs.V, 25, replace=False).astype(np.uint32), 0.5),
        (cs.disc(cs.at(0.9, 0.9), 0.1), 0.89999),                    # just under the limit
        (cs.disc(cs.at(0.9, 0.9), 0.1), 0.9),                        # at it
        (cs.disc(cs.at(0.2, 0.2), 0.2), np.inf),
    ]
    resumed = 0
    for ch, val in steps:
        cs.update(ch, val)
        got, ref = cs.replan(sf, sp)
        resumed += got["settled"] < ref["settled"]
    assert resumed >= 4, resumed
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_batch_replan_fixtures(api, oracle_mod, name):
    """the fuzz fixtures with deep cascades and a seed that pops after its neighbour, with the fixture's goal and four
    more: changes at several depths of the fixture goal's pop order"""
    pos, faces, vc, w, inv, sf0, sp0, cl = _fixture(name)
    cs = Case(api, oracle_mod, pos, faces, vc, 1.0, inv, cost_limit=cl, weights=w)
    sf, sp = cs.goals([(0.2, 0.3), (0.8, 0.7), (0.5, 0.5), (0.3, 0.8)])
    ok = np.array([inv is None or not inv[faces[f]].any() for f in sf])
    sf = np.concatenate([[sf0], sf[ok]]).astype(np.uint32); sp = np.concatenate([sp0[None], sp[ok]]).astype(np.float32)
    base, _ = cs.replan(sf, sp)
    d = base["dist"][0]
    fin = np.where(np.isfinite(d))[0]
    order = fin[np.argsort(d[fin], kind="stable")]
    for k, q in enumerate((0.1, 0.3, 0.5, 0.7, 0.9)):
        ch = order[int(q * (order.size - 1)):][:4]
        cs.update(ch, (vc[ch] + 0.05 * (k + 1)) % cl)
        cs.replan(sf, sp)
    cs.mm.close()


@pytest.mark.gpu
def test_batch_replan_goal_lists(api, oracle_mod):
    """goals added, dropped, reordered and duplicated between calls: rows follow their goals, duplicate rows are equal,
    and goals that stay resident resume"""
    rng = np.random.default_rng(7)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    sf, sp = cs.goals(_spread(10, rng))
    cs.replan(sf[:6], sp[:6])
    calls = [
        [5, 4, 3, 2, 1, 0],                   # reordered
        [0, 1, 2, 6, 7],                      # dropped and added
        [7, 7, 1, 0, 1, 8],                   # duplicates
        [9, 2, 8, 7],
        [7, 8, 9, 7],
    ]
    for k, idx in enumerate(calls):
        cs.update(cs.disc(cs.at(0.2 + 0.15 * k, 0.6), 0.1), 0.2 * k)
        got, ref = cs.replan(sf[idx], sp[idx])
        for i, j in [(i, j) for i in range(len(idx)) for j in range(i) if idx[i] == idx[j]]:
            for o in OUTS:
                assert _same(got[o][i], got[o][j]), o
        if k >= 2:
            assert got["settled"] < ref["settled"], k
    cs.mm.close()


@pytest.mark.gpu
def test_batch_replan_slot_cap(api, oracle_mod):
    """a cap of 3 slots and 8 goals: at most 3 goals resume, every row is exact; raising the cap resumes more goals"""
    rng = np.random.default_rng(9)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    sf, sp = cs.goals(_spread(8, rng))
    each = np.array([cs.settled(sf[i:i + 1], sp[i:i + 1]) for i in range(8)])
    hook = cs.mm.L.mnb_debug_set_batch_replan_slots
    assert hook(cs.mm._ctx, 3) == 0
    try:
        cs.replan(sf, sp)
        assert cs.mm.batch_replan_slots() == (3, 3)
        for k in range(2):
            cs.update(cs.disc(cs.at(0.95, 0.05 + 0.1 * k), 0.05), 0.8)
            got, ref = cs.replan(sf, sp)
            assert got["settled"] >= np.sort(each)[:5].sum()           # at least five goals ran whole
            assert got["settled"] < ref["settled"]
        capped = got["settled"]
        assert hook(cs.mm._ctx, 8) == 0
        cs.update(cs.disc(cs.at(0.95, 0.25), 0.05), 0.8)
        cs.replan(sf, sp)                                             # the five new slots fill
        assert cs.mm.batch_replan_slots() == (8, 8)
        cs.update(cs.disc(cs.at(0.95, 0.05), 0.05), 0.1)
        got, ref = cs.replan(sf, sp)
        assert got["settled"] < capped
        assert hook(cs.mm._ctx, 0) == 0                               # no slot: every goal whole
        cs.update(cs.disc(cs.at(0.95, 0.05), 0.05), 0.3)
        got, ref = cs.replan(sf, sp)
        assert got["settled"] == ref["settled"]
    finally:
        hook(cs.mm._ctx, -1)
    cs.mm.close()


@pytest.mark.gpu
def test_batch_replan_pool_overflow(api, oracle_mod):
    """resumed waves that run out of level pool (a test hook caps what they may add) run again as whole waves inside the
    kernel: every row is exact, and the retried waves are resident for the next call"""
    pos, faces, vc, w, inv, sf0, sp0, cl = _fixture("deep_cascade_planar")
    cs = Case(api, oracle_mod, pos, faces, vc, 1.0, inv, cost_limit=cl, weights=w)
    sf, sp = cs.goals([(0.3, 0.3), (0.7, 0.6)])
    sf = np.concatenate([[sf0], sf]).astype(np.uint32); sp = np.concatenate([sp0[None], sp]).astype(np.float32)
    hook = cs.mm.L.mnb_debug_set_replan_pool_room
    hook.argtypes = [C.c_void_p, C.c_uint32]
    base, ref = cs.replan(sf, sp)
    assert ref["deep_labels"] > 0
    d = base["dist"][0]
    fin = np.where(np.isfinite(d))[0]
    order = fin[np.argsort(d[fin], kind="stable")]
    ch = order[int(0.1 * order.size):][:3]
    assert hook(cs.mm._ctx, 1) == 0
    try:
        cs.update(ch, (vc[ch] + 0.1) % cl)
        cs.replan(sf, sp)
    finally:
        hook(cs.mm._ctx, 0)
    cs.update(ch, vc[ch])
    got, ref = cs.replan(sf, sp)
    assert got["settled"] < ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [1, 2, 4, 8])
def test_batch_replan_launch_forms(api, oracle_mod, cluster):
    """every cluster size of the batch kernel resumes exactly, with every output and with some of them"""
    rng = np.random.default_rng(12)
    pos, faces = _mesh("delaunay")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.6).astype(np.float32))
    cs.mm.set_tuning(0.0, cluster, 0)
    sf, sp = cs.goals(_spread(6, rng))
    cs.replan(sf, sp)
    for k, want in enumerate([OUTS, ("pred", "cutting_face"), ("dist",)]):
        cs.update(cs.disc(cs.at(0.4 + 0.15 * k, 0.5), 0.2), [np.inf, 0.2, 0.05][k])
        got, ref = cs.replan(sf, sp, want)
        assert got["settled"] < ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
def test_batch_replan_pointer_modes(api, oracle_mod):
    """device-pointer rows (a NULL output included) equal the host-pointer batch replan of a second context with the
    same history"""
    rng = np.random.default_rng(8)
    pos, faces = _mesh("terrain")
    costs = (rng.random(pos.shape[0]) * 0.5).astype(np.float32)
    a = Case(api, oracle_mod, pos, faces, costs)
    b = Case(api, oracle_mod, pos, faces, costs)
    sf, sp = a.goals(_spread(5, rng))
    n, V = sf.size, b.V
    on_gpu = not hasattr(b.mm.L, "mnb_emu_switch")
    for step in range(3):
        ch = a.disc(a.at(0.5 + 0.05 * step, 0.5), 0.12)
        a.update(ch, 0.6); b.update(ch, 0.6)
        got, _ = a.replan(sf, sp)
        pend = np.concatenate(b.pending); b.pending = []
        if on_gpu:
            import torch
            bufs = [torch.empty((n, V), dtype=t, device="cuda") for t in (torch.float32, torch.int32, torch.float32, torch.int32)]
            ptrs = [x.data_ptr() for x in bufs]
            back = lambda: [bufs[0].cpu().numpy(), bufs[1].cpu().numpy().view(np.uint32), bufs[2].cpu().numpy(), bufs[3].cpu().numpy()]
        else:
            # the interpreter runs a cluster launch as one forked process per CTA: what such a kernel writes reaches the
            # caller's memory only when that memory is shared
            bufs = [np.frombuffer(mmap.mmap(-1, 4 * n * V), t, n * V).reshape(n, V) for t in (np.float32, np.uint32, np.float32, np.int32)]
            ptrs = [x.ctypes.data for x in bufs]
            back = lambda: bufs
        if step == 2:
            ptrs[2] = 0                                               # a NULL output
        b.mm.use_device_pointers(True)
        try:
            rc = b.mm.cvp_batch_replan_dev(sf, sp, b.pl.cost_limit, pend, *ptrs)
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
def test_batch_replan_between_other_calls(api, oracle_mod):
    """mnb_cvp with back-tracking, mnb_cvp_replan, mnb_cvp_batch_fields, the Dijkstra field repair and the inflation repair
    between two batch replans: the store still resumes, and the batch replan disturbs neither the single replan's
    resident wave nor the last plan's back-tracking"""
    rng = np.random.default_rng(5)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    sf, sp = cs.goals(_spread(6, rng))
    _, rf, rp = centre_seed(pos, faces, (0.8, 0.75))
    sv = int(faces[sf[0]][0]); rv = int(faces[rf][0])
    dij = api.DijkstraMeshPlanner(cs.mm)
    infl = api.InflationLayer(cs.mm)
    cs.replan(sf, sp)
    single_pending = []
    cs.pl.waveFrontReplan(sf[0], sp[0], rf, [])
    plan = cs.pl.waveFrontPropagation(sf[1], sp[1], rf)
    path = cs.pl.backtrack(rp, rf)
    others = [
        lambda: cs.pl.backtrack(rp, rf),
        lambda: cs.pl.waveFrontReplan(sf[0], sp[0], rf, np.concatenate(single_pending)),
        lambda: cs.pl.waveFrontPropagationBatchFields(sf[:2], sp[:2]),
        lambda: dij.dijkstraBatchRepair([sv], [rv], *[dij.dijkstraBatch([sv])[k] for k in ("dist", "pred")]),
        lambda: infl.repairInflation(np.array([rv, sv], np.uint32)),
    ]
    for k, other in enumerate(others):
        ch = cs.disc(cs.at(0.6, 0.62), 0.08 + 0.01 * k)
        cs.update(ch, 0.3 + 0.05 * k)
        single_pending.append(ch)
        res = other()
        if k == 1:
            single_pending = []
            assert res["settled"] < cs.pl.waveFrontPropagation(sf[0], sp[0], rf)["settled"]   # the single replan resumed
            plan = cs.pl.waveFrontPropagation(sf[1], sp[1], rf)
            path = cs.pl.backtrack(rp, rf)
        got, ref = cs.replan(sf, sp)
        assert got["settled"] < ref["settled"], k
        if k != 1:
            # the fresh batch ran after the replan: the last plan's back-tracking still gives its path
            bt = cs.pl.backtrack(rp, rf)
            assert bt["outcome"] == path["outcome"] and _same(bt["positions"], path["positions"]), k
    assert plan["outcome"] == 0
    cs.mm.close()


def _raw(mm, sf, sp, changed, outs, changed_ptr=True, cost_limit=1.0):
    sf = np.ascontiguousarray(sf, np.uint32); sp = np.ascontiguousarray(sp, np.float32); ch = np.ascontiguousarray(changed, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    return mm.L.mnb_cvp_batch_replan(mm._ctx, sf.size, p(sf), p(sp), float(cost_limit), ch.size, p(ch) if changed_ptr else None,
                                     *[p(o) for o in outs])


@pytest.mark.gpu
def test_batch_replan_arguments(api, oracle_mod):
    """n == 0, all outputs NULL, a changed vertex >= V or a NULL changed list with n > 0 -> MNB_E_ARG (-1); no costs ->
    MNB_E_STATE (-3); a seed face >= F -> INVALID_START (52); nothing is written in any of these"""
    pos, faces = mesh_case(16, True)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    V, F = om.V, faces.shape[0]
    sf = np.array([5, 40], np.uint32); sp = pos[faces[sf]].mean(1)
    outs = [np.full((2, V), 7, t) for t in (np.float32, np.uint32, np.float32, np.int32)]
    untouched = lambda: all((o == 7).all() for o in outs)
    assert _raw(mm, sf, sp, [1], outs) == -3 and untouched()
    mm.setCosts(np.zeros(V, np.float32), om.edge_distances())
    assert _raw(mm, sf[:0], sp[:0], [1], outs) == -1 and untouched()
    assert _raw(mm, sf, sp, [1], [None] * 4) == -1
    assert _raw(mm, sf, sp, [1, V], outs) == -1 and untouched()
    assert _raw(mm, sf, sp, [1], outs, changed_ptr=False) == -1 and untouched()
    assert _raw(mm, [5, F], sp, [1], outs) == 52 and untouched()
    assert _raw(mm, sf, sp, [], outs) == 0 and not untouched()
    ref = api.CVPMeshPlanner(mm).waveFrontPropagationBatchFields(sf, sp)
    for k, o in zip(OUTS, outs):
        assert _same(o, ref[k]), k
    mm.close()


@pytest.mark.gpu
def test_batch_replan_release(api, oracle_mod):
    """after mnb_cvp_batch_replan_release the next call runs whole waves; on the interpreter the allocated device bytes
    drop by the store's size"""
    rng = np.random.default_rng(6)
    pos, faces = _mesh("terrain")
    cs = Case(api, oracle_mod, pos, faces, (rng.random(pos.shape[0]) * 0.5).astype(np.float32))
    sf, sp = cs.goals(_spread(4, rng))
    L = cs.mm.L
    emu = hasattr(L, "mnb_emu_allocated_bytes")
    if emu:
        L.mnb_emu_allocated_bytes.restype = C.c_size_t
    cs.replan(sf, sp)
    before = L.mnb_emu_allocated_bytes() if emu else 0
    assert cs.mm.batch_replan_slots() == (4, 4)
    assert L.mnb_cvp_batch_replan_release(cs.mm._ctx) == 0
    assert cs.mm.batch_replan_slots() == (0, 0)
    if emu:
        V = cs.V
        slot = 36 * V + 4 * max(65536, 2 * V) + 16
        assert before - L.mnb_emu_allocated_bytes() >= 4 * slot
    cs.update(cs.disc(cs.at(0.5, 0.5), 0.1), 0.4)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] == ref["settled"]
    cs.update(cs.disc(cs.at(0.5, 0.5), 0.1), 0.2)
    got, ref = cs.replan(sf, sp)
    assert got["settled"] < ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
def test_batch_replan_cancel(api, oracle_mod):
    """mnb_cancel from another thread -> CANCELED (51); the store is dropped: the next call runs whole waves"""
    pos, faces = mesh_case(300, True)
    cs = Case(api, oracle_mod, pos, faces)
    cs.mm.set_tuning(0.002, 1, 0)                                    # narrow band on one CTA per wave: slow waves
    rng = np.random.default_rng(2)
    sf, sp = cs.goals(_spread(32, rng))
    cs.replan(sf, sp, ("dist",))
    allv = np.arange(cs.V, dtype=np.uint32)                          # T0 before the seeds: whole waves in the slots
    t0 = time.perf_counter(); whole = cs.pl.waveFrontReplanBatch(sf, sp, allv, want=("dist",)); t_full = time.perf_counter() - t0
    assert whole["outcome"] == 0 and t_full > 0.05, t_full
    outcomes = []
    t = threading.Thread(target=lambda: outcomes.append(cs.pl.waveFrontReplanBatch(sf, sp, allv, want=("dist",))["outcome"]))
    t.start(); time.sleep(0.3 * t_full); cs.mm.cancel(); t.join()
    assert outcomes == [51]
    assert cs.mm.batch_replan_slots()[1] == 0
    got, ref = cs.replan(sf, sp, ("dist",))
    assert got["settled"] == ref["settled"]
    cs.mm.close()


@pytest.mark.gpu
def test_batch_replan_large(api, oracle_mod):
    """1 M-vertex terrain, 64 goals, one disc change: every row is exact and the re-run share is below the fresh batch's"""
    pos, faces = mesh_case(1000, True)
    cs = Case(api, oracle_mod, pos, faces)
    rng = np.random.default_rng(1)
    sf, sp = cs.goals(_spread(64, rng))
    want = ("dist", "pred")
    cs.replan(sf, sp, want)
    cs.update(cs.disc(cs.at(0.7, 0.4), 0.3), 0.8)
    got, ref = cs.replan(sf, sp, want)
    print(f"settled {got['settled']} of {ref['settled']}, kernel {got['kernel_ms']:.1f} ms against {ref['kernel_ms']:.1f} ms")
    assert got["settled"] < ref["settled"]
    cs.mm.close()


@pytest.mark.parametrize("shuffle, expr", [
    (None, "not large and not cancel"),
    ("5", "first_call or fixtures or launch_forms or overflow or goal_lists or slot_cap or (changes and terrain)"),
])
def test_cvp_batch_replan_on_the_cpu_interpreter(shuffle, expr):
    """the GPU tests above (minus the 1 M-vertex and the cancel test) with the kernels compiled by g++ against tests/emu,
    on 4 emulated SMs, in the default warp order; a part of them again in a randomised one"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    env = dict(os.environ, MNB_EMU_SMS="4", **({"MNB_EMU_SHUFFLE": shuffle} if shuffle else {}))
    r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider", "-k", expr],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=560)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"shuffle {shuffle}:\n{tail}"
