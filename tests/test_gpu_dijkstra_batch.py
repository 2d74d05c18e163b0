"""Batched full-field Dijkstra (mnb_dijkstra_batch / DijkstraMeshPlanner.dijkstraBatch): every row against the oracle's
DijkstraMeshPlanner::dijkstra (dijkstra_mesh_planner.cpp:217-398, robot vertex -1) -- distances bit for bit as uint32,
predecessors exactly -- and against mnb_dijkstra with the same seed.  The GPU tests run with -m gpu on an H100; the last
test replays them on the CPU interpreter of the kernels (tests/emu)."""
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


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _map(api, oracle_mod, n, terrain=True, costs=None, factor=0.0, invalid=None, seed=42):
    pos, faces = mesh_case(n, terrain, seed)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    ed = om.edge_distances()
    vc = np.zeros(om.V, np.float32) if costs is None else costs.astype(np.float32)
    w = om.edge_weights(vc, ed, factor)
    mm.setCosts(vc, w, invalid)
    return pos, faces, om, mm, ed, vc, w


def _check_rows(om, w, vc, seeds, got, invalid=None, cost_limit=1.0, rows=None):
    for k in (range(len(seeds)) if rows is None else rows):
        ref = om.dijkstra(w, vc, int(seeds[k]), invalid=invalid, cost_limit=cost_limit)
        if got["dist"] is not None:
            assert (got["dist"][k].view(np.uint32) == ref["dist"].view(np.uint32)).all(), f"row {k} (seed {seeds[k]}): dist"
        if got["pred"] is not None:
            assert (got["pred"][k] == ref["pred"]).all(), f"row {k} (seed {seeds[k]}): pred"


def _raw(mm, seeds, want_dist=True, want_pred=True, cost_limit=1.0):
    """mnb_dijkstra_batch in host-pointer mode with either output optional"""
    sv = np.ascontiguousarray(seeds, dtype=np.uint32)
    dist = np.full((sv.size, mm.V), 7.0, np.float32) if want_dist else None
    pred = np.full((sv.size, mm.V), 7, np.uint32) if want_pred else None
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = mm.L.mnb_dijkstra_batch(mm._ctx, sv.size, p(sv), float(cost_limit), p(dist), p(pred))
    return rc, dist, pred


def _walk(pred, v):
    path = [int(v)]
    while int(pred[path[-1]]) != path[-1]:
        path.append(int(pred[path[-1]]))
        assert len(path) <= pred.size
    return path


def _wall_costs(pos, rng):
    """cost regions over the cost limit, and a +inf wall that leaves the far side of the map unreached"""
    c = np.where(rng.random(pos.shape[0]) < 0.05, 1.5, rng.random(pos.shape[0]) * 0.8).astype(np.float32)
    c[(pos[:, 0] > 5.0) & (pos[:, 0] < 5.4)] = np.inf
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
def test_dijkstra_batch_parity(api, oracle_mod, factor):
    rng = np.random.default_rng(11)
    pos, faces = mesh_case(100, True)
    costs = _wall_costs(pos, rng)
    invalid = (rng.random(pos.shape[0]) < 0.01).astype(np.uint8)
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 100, costs=costs, factor=factor, invalid=invalid)
    seeds = rng.choice(om.V, 24, replace=False).astype(np.uint32)
    pl = api.DijkstraMeshPlanner(mm)
    got = pl.dijkstraBatch(seeds)
    assert got["outcome"] == 0 and got["dist"].shape == (24, om.V) and got["pred"].shape == (24, om.V)
    _check_rows(om, w, vc, seeds, got, invalid=invalid)
    unreached = np.isinf(got["dist"]).sum(1)
    assert (unreached > om.V // 3).all(), "the wall leaves part of the map unreached"
    # stats of the whole batch: every finite label but the seed's is settled once by the round loop
    assert got["settled"] == int(np.isfinite(got["dist"]).sum()) - len(seeds) and got["rounds"] > 0 and got["kernel_launches"] == 1
    for k, s in enumerate(seeds):
        one = pl.dijkstra(int(s))
        assert (one["dist"].view(np.uint32) == got["dist"][k].view(np.uint32)).all() and (one["pred"] == got["pred"][k]).all()
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_edge_cases(api, oracle_mod):
    """seed on the border, on an invalid vertex, over the cost limit, duplicate seeds; a disconnected mesh; one face"""
    rng = np.random.default_rng(5)
    pos, faces = mesh_case(60, True)
    costs = np.where(rng.random(pos.shape[0]) < 0.1, 1.5, 0.3).astype(np.float32)
    invalid = (rng.random(pos.shape[0]) < 0.02).astype(np.uint8)
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 60, costs=costs, factor=1.0, invalid=invalid)
    inv_v = int(np.where(invalid)[0][0]); over_v = int(np.where((vc > 1.0) & (invalid == 0))[0][0])
    v, _, _ = centre_seed(pos, faces)
    seeds = np.array([0, inv_v, over_v, v, v, 59, inv_v], np.uint32)
    got = api.DijkstraMeshPlanner(mm).dijkstraBatch(seeds)
    assert got["outcome"] == 0
    _check_rows(om, w, vc, seeds, got, invalid=invalid)
    assert np.isfinite(got["dist"][2]).sum() == 1 and (got["dist"][3].view(np.uint32) == got["dist"][4].view(np.uint32)).all()
    mm.close()
    # two components: the other one stays +inf with every vertex its own predecessor
    pos1, faces1 = mesh_case(20, False)
    pos = np.concatenate([pos1, pos1 + np.array([10.0, 0, 0], np.float32)])
    faces = np.concatenate([faces1, faces1 + len(pos1)]).astype(np.uint32)
    om = oracle_mod.OracleMesh(pos, faces); mm = api.MeshMap(pos, faces)
    ed = om.edge_distances(); vc = np.zeros(om.V, np.float32); mm.setCosts(vc, ed)
    seeds = np.array([5, len(pos1) + 7, 5], np.uint32)
    got = api.DijkstraMeshPlanner(mm).dijkstraBatch(seeds)
    _check_rows(om, ed, vc, seeds, got)
    n1 = len(pos1)
    assert np.isinf(got["dist"][0][n1:]).all() and (got["pred"][0][n1:] == np.arange(n1, om.V)).all()
    assert np.isinf(got["dist"][1][:n1]).all() and (got["pred"][1][:n1] == np.arange(n1)).all()
    mm.close()
    tri_pos = np.array([[0, 0, 0], [0.5, 0, 0], [0, 0.5, 0]], np.float32); tri = np.array([[0, 1, 2]], np.uint32)
    om = oracle_mod.OracleMesh(tri_pos, tri); mm = api.MeshMap(tri_pos, tri)
    ed = om.edge_distances(); mm.setCosts(np.zeros(3, np.float32), ed)
    got = api.DijkstraMeshPlanner(mm).dijkstraBatch([0, 1, 2, 0])
    assert got["dist"][0].tolist() == [0.0, 0.5, 0.5] and got["pred"][0].tolist() == [0, 0, 0]
    _check_rows(om, ed, np.zeros(3, np.float32), [0, 1, 2, 0], got)
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_counts_and_tuning(api, oracle_mod):
    """one and three seeds (clusters of CTAs per wavefront), more seeds than wavefronts in flight, and rows that do not
    depend on the band width or the cluster size"""
    rng = np.random.default_rng(3)
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 60, costs=(rng.random(3600) * 0.8), factor=1.0)
    pl = api.DijkstraMeshPlanner(mm)
    seeds = rng.choice(om.V, 5, replace=False).astype(np.uint32)
    base = pl.dijkstraBatch(seeds)
    _check_rows(om, w, vc, seeds, base)
    for n in (1, 3):
        got = pl.dijkstraBatch(seeds[:n])
        _check_rows(om, w, vc, seeds[:n], got)
    for delta, cluster in ((0.0, 1), (0.0, 4), (0.02, 0), (1e30, 0)):
        mm.set_tuning(delta, cluster, 0)
        got = pl.dijkstraBatch(seeds)
        assert (got["dist"].view(np.uint32) == base["dist"].view(np.uint32)).all(), (delta, cluster)
        assert (got["pred"] == base["pred"]).all(), (delta, cluster)
    mm.close()
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 20, costs=(rng.random(400) * 0.8), factor=1.0)
    seeds = rng.integers(0, om.V, 600).astype(np.uint32)
    got = api.DijkstraMeshPlanner(mm).dijkstraBatch(seeds)
    assert got["outcome"] == 0
    ref = {}
    for k, s in enumerate(seeds):
        if int(s) not in ref:
            ref[int(s)] = om.dijkstra(w, vc, int(s))
        r = ref[int(s)]
        assert (got["dist"][k].view(np.uint32) == r["dist"].view(np.uint32)).all() and (got["pred"][k] == r["pred"]).all(), k
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_output_modes(api, oracle_mod):
    """dist only, pred only, both; device pointers give the same bytes as host pointers"""
    rng = np.random.default_rng(8)
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 50, costs=(rng.random(2500) * 0.8), factor=1.0)
    seeds = rng.choice(om.V, 6, replace=False).astype(np.uint32)
    rc, dist, pred = _raw(mm, seeds)
    assert rc == 0
    _check_rows(om, w, vc, seeds, dict(dist=dist, pred=pred))
    rc, d_only, none = _raw(mm, seeds, want_pred=False)
    assert rc == 0 and none is None and (d_only.view(np.uint32) == dist.view(np.uint32)).all()
    rc, none, p_only = _raw(mm, seeds, want_dist=False)
    assert rc == 0 and none is None and (p_only == pred).all()
    # decided by the loaded library: the CPU interpreter (it exports its fiber switch) cannot dereference device pointers
    on_gpu = not hasattr(mm.L, "mnb_emu_switch")
    if on_gpu:
        import torch
        d_dist = torch.full((seeds.size, om.V), 7.0, dtype=torch.float32, device="cuda")
        d_pred = torch.full((seeds.size, om.V), 7, dtype=torch.int32, device="cuda")
        ptr = lambda t: t.data_ptr(); back = lambda t: t.cpu().numpy()
    else:
        d_dist = np.full((seeds.size, om.V), 7.0, np.float32); d_pred = np.full((seeds.size, om.V), 7, np.uint32)
        ptr = lambda a: a.ctypes.data; back = lambda a: a
    mm.use_device_pointers(True)
    try:
        assert mm.dijkstra_batch_dev(seeds, 1.0, ptr(d_dist), ptr(d_pred)) == 0
        if on_gpu:
            torch.cuda.synchronize()
        assert (back(d_dist).view(np.uint32) == dist.view(np.uint32)).all() and (back(d_pred).view(np.uint32) == pred).all()
        if on_gpu:
            d_dist.fill_(7.0)
        else:
            d_dist[:] = 7.0
        assert mm.dijkstra_batch_dev(seeds, 1.0, ptr(d_dist), 0) == 0
        if on_gpu:
            torch.cuda.synchronize()
        assert (back(d_dist).view(np.uint32) == dist.view(np.uint32)).all()
    finally:
        mm.use_device_pointers(False)
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_arguments_and_state(api, oracle_mod):
    """n == 0 and both outputs NULL -> MNB_E_ARG (-1); a seed >= V -> INVALID_START (52) with nothing written; no costs
    installed -> MNB_E_STATE (-3)"""
    pos, faces = mesh_case(30, True)
    mm = api.MeshMap(pos, faces)
    rc, dist, pred = _raw(mm, [3, 4])
    assert rc == -3
    om = oracle_mod.OracleMesh(pos, faces); ed = om.edge_distances(); mm.setCosts(np.zeros(om.V, np.float32), ed)
    rc, dist, pred = _raw(mm, [3, om.V, 4])
    assert rc == 52 and (dist == 7.0).all() and (pred == 7).all()
    rc, _, _ = _raw(mm, [3], want_dist=False, want_pred=False)
    assert rc == -1
    dist = np.empty((1, om.V), np.float32)
    assert mm.L.mnb_dijkstra_batch(mm._ctx, 0, np.zeros(1, np.uint32).ctypes.data_as(C.c_void_p), 1.0,
                                   dist.ctypes.data_as(C.c_void_p), None) == -1
    assert mm.L.mnb_dijkstra_batch(mm._ctx, 1, None, 1.0, dist.ctypes.data_as(C.c_void_p), None) == -1
    rc, dist, pred = _raw(mm, [3])
    assert rc == 0
    _check_rows(om, ed, np.zeros(om.V, np.float32), [3], dict(dist=dist, pred=pred))
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_after_other_calls(api, oracle_mod):
    """the batch reads the current weights after mnb_update_vertex_costs; it leaves the last mnb_cvp's back-tracking
    field and the last inflation's labels alone; single plans after it stay bit-exact"""
    rng = np.random.default_rng(21)
    costs = (0.45 + 0.45 * np.sin(3.0 * mesh_case(80, True)[0][:, 0])).astype(np.float32)
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 80, costs=costs, factor=1.0)
    dpl = api.DijkstraMeshPlanner(mm); cpl = api.CVPMeshPlanner(mm)
    seeds = rng.choice(om.V, 8, replace=False).astype(np.uint32)
    _check_rows(om, w, vc, seeds, dpl.dijkstraBatch(seeds))
    changed = np.unique(rng.choice(om.V, 300, replace=False)).astype(np.uint32)
    mm.layerChanged(changed, (rng.random(changed.size) * 0.9).astype(np.float32), 1.0)
    vc2, w2 = mm.costs()
    assert (w2 != w).any()
    _check_rows(om, w2, vc2, seeds, dpl.dijkstraBatch(seeds))
    sv, sf, sp = centre_seed(pos, faces, (0.2, 0.25))
    cfull = cpl.waveFrontPropagation(sf, sp)
    # mnb_cvp -> batch -> mnb_cvp_backtrack / mnb_vector_map(pred = NULL): the same as without the batch
    rv, rf, rp = centre_seed(pos, faces, (0.8, 0.7))
    vec = lambda: (mm.L.mnb_vector_map(mm._ctx, None, None, None, out.ctypes.data_as(C.c_void_p)), out.copy())[1]
    out = np.empty((om.V, 3), np.float32)
    c0 = cpl.waveFrontPropagation(sf, sp, rf)
    assert c0["outcome"] == 0
    bt0 = cpl.backtrack(rp, rf); vm0 = vec()
    cpl.waveFrontPropagation(sf, sp, rf)
    dpl.dijkstraBatch(seeds)
    bt1 = cpl.backtrack(rp, rf); vm1 = vec()
    assert bt0["outcome"] == bt1["outcome"] == 0 and len(bt0["positions"]) > 10
    assert (bt0["positions"].view(np.uint32) == bt1["positions"].view(np.uint32)).all() and (bt0["faces"] == bt1["faces"]).all()
    assert (vm0.view(np.uint32) == vm1.view(np.uint32)).all()
    # the last inflation's vector field can still be derived after a batch
    infl = api.InflationLayer(mm)
    infl.waveCostInflation(np.array([sv, rv], np.uint32))
    dpl.dijkstraBatch(seeds[:2])
    assert infl.vectorMap().shape == (om.V, 3)
    # single plans after the batch
    one = dpl.dijkstra(int(seeds[0]))
    ref = om.dijkstra(w2, vc2, int(seeds[0]))
    assert (one["dist"].view(np.uint32) == ref["dist"].view(np.uint32)).all() and (one["pred"] == ref["pred"]).all()
    c2 = cpl.waveFrontPropagation(sf, sp)
    for k in ("dist", "pred", "direction", "cutting_face"):
        assert (c2[k].view(np.uint32) == cfull[k].view(np.uint32)).all(), k
    oc = om.cvp(w2, vc2, sf, sp)
    fin = np.isfinite(oc["dist"])
    assert (np.isfinite(c2["dist"]) == fin).all()
    assert (np.abs(c2["dist"][fin].astype(np.float64) - oc["dist"][fin]) <= 1e-4 * np.maximum(oc["dist"][fin], 1e-30)).all()
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_rows_feed_vector_map_and_paths(api, oracle_mod):
    """a predecessor row is a DijkstraMeshPlanner::computeVectorMap input (:189-209) and the path to its seed from any
    robot vertex (:367-373)"""
    rng = np.random.default_rng(4)
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 90, costs=(rng.random(8100) * 0.8).astype(np.float32), factor=1.0)
    pl = api.DijkstraMeshPlanner(mm)
    seeds = np.array([centre_seed(pos, faces, uv)[0] for uv in ((0.3, 0.3), (0.7, 0.4), (0.5, 0.8))], np.uint32)
    got = pl.dijkstraBatch(seeds)
    for k in range(len(seeds)):
        ref = om.dijkstra_vector_map(got["pred"][k]); vm = pl.computeVectorMap(got["pred"][k])
        assert (np.isnan(ref) == np.isnan(vm)).all()
        ok = ~np.isnan(ref)
        assert (vm[ok].view(np.uint32) == ref[ok].view(np.uint32)).all()
    for robot_uv in ((0.9, 0.1), (0.1, 0.9)):
        rv = centre_seed(pos, faces, robot_uv)[0]
        for k, s in enumerate(seeds):
            single = pl.dijkstra(int(s), int(rv))
            assert single["outcome"] == 0
            path = _walk(got["pred"][k], rv)
            assert path == _walk(single["pred"], rv) and path[-1] == int(s)
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_cancel(api, oracle_mod):
    """mnb_cancel from another thread during a batch -> CANCELED (51); the persistent groups take no new seeds, and the
    next call succeeds"""
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 120)
    mm.set_tuning(0.005, 1, 0)         # narrow band: many rounds per wavefront
    pl = api.DijkstraMeshPlanner(mm)
    rng = np.random.default_rng(2)
    n = 8
    while True:                        # grow the batch until it takes long enough for the cancel to land inside it
        seeds = rng.integers(0, om.V, n).astype(np.uint32)
        t0 = time.perf_counter(); full = pl.dijkstraBatch(seeds, want_pred=False); t_full = time.perf_counter() - t0
        assert full["outcome"] == 0
        if t_full > 0.2 or n >= 16384:
            break
        n *= 4
    assert t_full > 0.05, t_full
    outcomes = []

    def run():
        t1 = time.perf_counter(); o = pl.dijkstraBatch(seeds, want_pred=False)["outcome"]; outcomes.append((o, time.perf_counter() - t1))
    t = threading.Thread(target=run)
    t.start(); time.sleep(0.25 * t_full); mm.cancel(); t.join()
    assert outcomes[0][0] == 51, outcomes
    assert outcomes[0][1] < 0.85 * t_full, (outcomes, t_full)
    got = pl.dijkstraBatch(seeds[:2])
    assert got["outcome"] == 0
    _check_rows(om, w, vc, seeds[:2], got)
    mm.close()


@pytest.mark.gpu
def test_dijkstra_batch_large_mesh(api, oracle_mod):
    """1 M-vertex terrain, 64 seeds, 4 rows against the oracle"""
    from mesh_navigation_b200 import synth
    pos, faces, om, mm, ed, vc, w = _map(api, oracle_mod, 1000)
    seeds = synth.batch_goal_vertices(om.V, 64, seed=1234).astype(np.uint32)
    got = api.DijkstraMeshPlanner(mm).dijkstraBatch(seeds)
    assert got["outcome"] == 0 and np.isfinite(got["dist"]).all()
    _check_rows(om, w, vc, seeds, got, rows=[0, 21, 42, 63])
    mm.close()


def test_dijkstra_batch_on_the_cpu_interpreter():
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
