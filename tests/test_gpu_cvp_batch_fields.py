"""Batched CVP vector fields (mnb_cvp_batch_fields / CVPMeshPlanner.waveFrontPropagationBatchFields): every row of the
potential, predecessor, direction and cutting-face outputs against mnb_cvp with the same goal (robot face -1) bit for bit,
and against the oracle's CVPMeshPlanner::waveFrontPropagation (cvp_mesh_planner.cpp:651-886) -- potentials bit for bit,
predecessors and cutting faces exactly, directions bit for bit on the CPU interpreter and on the GPU at most one float ulp
apart on fewer than 1e-4 of the vertices (CUDA's and glibc's double acos may differ in the last bit).  The GPU tests run with -m gpu on an H100; the last test
replays them on the CPU interpreter of the kernels (tests/emu)."""
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
KEYS = ("dist", "pred", "direction", "cutting_face")


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _fuzz_case(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", f"fuzz_{name}.npz"))
    inv = d["inv"] if d["inv"].size else None
    return d["pos"], d["faces"], d["vc"], d["w"], inv, int(d["sf"]), d["sp"], float(d["cl"])


def _map(api, oracle_mod, n, costs=None, factor=0.0, invalid=None):
    pos, faces = mesh_case(n, True)
    om = oracle_mod.OracleMesh(pos, faces)
    mm = api.MeshMap(pos, faces)
    ed = om.edge_distances()
    vc = np.zeros(om.V, np.float32) if costs is None else costs.astype(np.float32)
    w = om.edge_weights(vc, ed, factor)
    mm.setCosts(vc, w, invalid)
    return pos, faces, om, mm, vc, w


def _goals(pos, faces, sfs):
    sfs = np.asarray(sfs, np.uint32)
    return sfs, np.stack([pos[faces[f]].mean(0) for f in sfs]).astype(np.float32)


def _same(a, b):
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def _direction_ok(got, ref):
    """directions against the oracle's: bit for bit on the CPU interpreter (its acos is the oracle's); on the GPU at most
    one float ulp apart, on fewer than 1e-4 of the vertices"""
    from mesh_navigation_b200 import _lib
    line = lambda x: (lambda i: np.where(i < 0, -(i & 0x7FFFFFFF), i))(np.asarray(x, np.float32).view(np.int32).astype(np.int64))
    u = np.abs(line(got) - line(ref))
    if _lib.LIB_PATH.endswith("libmeshnav_emu.so"):
        return (u == 0).all()
    return u.max() <= 1 and np.count_nonzero(u) < 1e-4 * u.size


def _check_oracle(om, w, vc, sfs, sps, got, invalid=None, cost_limit=1.0, rows=None):
    for k in (range(len(sfs)) if rows is None else rows):
        ref = om.cvp(w, vc, int(sfs[k]), sps[k], invalid=invalid, cost_limit=cost_limit)
        if got["dist"] is not None:
            assert _same(got["dist"][k], ref["dist"]), f"row {k} (face {sfs[k]}): dist"
        if got["pred"] is not None:
            assert (got["pred"][k] == ref["pred"]).all(), f"row {k}: pred"
        if got["cutting_face"] is not None:
            assert (got["cutting_face"][k] == ref["cutting_face"]).all(), f"row {k}: cutting_face"
        if got["direction"] is not None:
            assert _direction_ok(got["direction"][k], ref["direction"]), f"row {k}: direction"


def _check_single(pl, sfs, sps, got, rows=None):
    """row k == mnb_cvp(seed k, robot face -1), every requested output bit for bit"""
    for k in (range(len(sfs)) if rows is None else rows):
        one = pl.waveFrontPropagation(int(sfs[k]), sps[k])
        assert one["outcome"] == 0
        for key in KEYS:
            if got[key] is not None:
                assert _same(got[key][k], one[key]), f"row {k} (face {sfs[k]}): {key}"


def _raw(mm, sfs, sps, want=KEYS, cost_limit=1.0):
    """mnb_cvp_batch_fields in host-pointer mode, outputs pre-filled with 7"""
    sf = np.ascontiguousarray(sfs, dtype=np.uint32); sp = np.ascontiguousarray(sps, dtype=np.float32).reshape(-1, 3)
    kinds = dict(dist=np.float32, pred=np.uint32, direction=np.float32, cutting_face=np.int32)
    out = {k: (np.full((sf.size, mm.V), 7, t) if k in want else None) for k, t in kinds.items()}
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = mm.L.mnb_cvp_batch_fields(mm._ctx, sf.size, p(sf), p(sp), float(cost_limit), p(out["dist"]), p(out["pred"]),
                                   p(out["direction"]), p(out["cutting_face"]))
    return rc, out


def _wall_costs(pos, rng):
    """cost regions over the cost limit, and a +inf wall that leaves the far side of the map unreached"""
    c = np.where(rng.random(pos.shape[0]) < 0.05, 1.5, rng.random(pos.shape[0]) * 0.8).astype(np.float32)
    c[(pos[:, 0] > 3.0) & (pos[:, 0] < 3.4)] = np.inf
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
def test_cvp_batch_fields_parity(api, oracle_mod, factor):
    rng = np.random.default_rng(11)
    pos, faces = mesh_case(60, True)
    costs = _wall_costs(pos, rng)
    invalid = (rng.random(pos.shape[0]) < 0.01).astype(np.uint8)
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 60, costs=costs, factor=factor, invalid=invalid)
    sfs, sps = _goals(pos, faces, rng.choice(om.F, 12, replace=False))
    pl = api.CVPMeshPlanner(mm)
    got = pl.waveFrontPropagationBatchFields(sfs, sps)
    assert got["outcome"] == 0 and got["kernel_launches"] == 1 and got["rounds"] > 0
    for key in KEYS:
        assert got[key].shape == (12, om.V)
    _check_oracle(om, w, vc, sfs, sps, got, invalid=invalid)
    _check_single(pl, sfs, sps, got)
    assert (np.isinf(got["dist"]).sum(1) > 0).all(), "the wall leaves part of the map unreached"
    unreached = np.isinf(got["dist"])
    assert (got["pred"][unreached] == np.nonzero(unreached)[1]).all() and (got["cutting_face"][unreached] == -1).all()
    assert (got["direction"][unreached] == 0).all()
    mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour"])
def test_cvp_batch_fields_hard_cases(api, oracle_mod, name):
    """cascades of any depth, cost-limit walls, invalid vertices and seeds that pop late, at every cluster size and
    several band widths: the epilogue of each wavefront reads the level pool of its own workspace group"""
    pos, faces, vc, w, inv, sf, sp, cl = _fuzz_case(name)
    om = oracle_mod.OracleMesh(pos, faces)
    rng = np.random.default_rng(5)
    sfs, sps = _goals(pos, faces, np.concatenate([[sf], rng.integers(0, om.F, 4)]))
    sps[0] = sp
    mm = api.MeshMap(pos, faces)
    mm.setCosts(vc, w, inv)
    pl = api.CVPMeshPlanner(mm, cost_limit=cl)
    singles = [pl.waveFrontPropagation(int(sfs[k]), sps[k]) for k in range(len(sfs))]
    refs = [om.cvp(w, vc, int(sfs[k]), sps[k], invalid=inv, cost_limit=cl) for k in range(len(sfs))]
    for cluster, delta in ((1, 0.3), (2, 0.1), (4, 1.8), (8, 0.3), (1, 0.05)):
        mm.set_tuning(delta, cluster, 0)
        got = pl.waveFrontPropagationBatchFields(sfs, sps)
        assert got["outcome"] == 0
        for k in range(len(sfs)):
            for key in KEYS:
                assert _same(got[key][k], singles[k][key]), (cluster, delta, k, key)
            assert _same(got["dist"][k], refs[k]["dist"]), (cluster, delta, k)
            assert (got["pred"][k] == refs[k]["pred"]).all() and (got["cutting_face"][k] == refs[k]["cutting_face"]).all(), (cluster, delta, k)
            assert _direction_ok(got["direction"][k], refs[k]["direction"]), (cluster, delta, k)
        if name.startswith("deep_cascade"):
            assert got["deep_labels"] >= singles[0]["deep_labels"] > 0          # counted by the per-wave epilogue
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_edge_cases(api, oracle_mod):
    """a seed face with a vertex over the cost limit, one with an invalid vertex, duplicate goals; a disconnected mesh;
    a one-face mesh"""
    rng = np.random.default_rng(5)
    pos, faces = mesh_case(40, True)
    costs = np.where(rng.random(pos.shape[0]) < 0.1, 1.5, 0.3).astype(np.float32)
    invalid = (rng.random(pos.shape[0]) < 0.02).astype(np.uint8)
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 40, costs=costs, factor=1.0, invalid=invalid)
    over_f = int(np.where((vc[faces] > 1.0).any(1) & (invalid[faces] == 0).all(1))[0][0])
    inv_f = int(np.where(invalid[faces].any(1))[0][0])
    _, cf, _ = centre_seed(pos, faces)
    sfs, sps = _goals(pos, faces, [over_f, inv_f, cf, cf, 0, over_f])
    pl = api.CVPMeshPlanner(mm)
    got = pl.waveFrontPropagationBatchFields(sfs, sps)
    assert got["outcome"] == 0
    _check_oracle(om, w, vc, sfs, sps, got, invalid=invalid)
    _check_single(pl, sfs, sps, got)
    for key in KEYS:
        assert _same(got[key][2], got[key][3]) and _same(got[key][0], got[key][5]), key
    seeds = faces[cf]
    assert (got["pred"][2][seeds] == seeds).all() and (got["cutting_face"][2][seeds] == cf).all() and (got["direction"][2][seeds] == 0).all()
    mm.close()
    # two components: the other one gets +inf, self, 0 and -1
    pos1, faces1 = mesh_case(20, False)
    pos = np.concatenate([pos1, pos1 + np.array([10.0, 0, 0], np.float32)])
    faces = np.concatenate([faces1, faces1 + len(pos1)]).astype(np.uint32)
    om = oracle_mod.OracleMesh(pos, faces); mm = api.MeshMap(pos, faces)
    ed = om.edge_distances(); vc = np.zeros(om.V, np.float32); mm.setCosts(vc, ed)
    n1, f1 = len(pos1), len(faces1)
    sfs, sps = _goals(pos, faces, [5, f1 + 7, 5])
    got = api.CVPMeshPlanner(mm).waveFrontPropagationBatchFields(sfs, sps)
    _check_oracle(om, ed, vc, sfs, sps, got)
    for k, other in ((0, np.arange(n1, om.V)), (1, np.arange(n1))):
        assert np.isinf(got["dist"][k][other]).all() and (got["pred"][k][other] == other).all()
        assert (got["direction"][k][other] == 0).all() and (got["cutting_face"][k][other] == -1).all()
    mm.close()
    tri_pos = np.array([[0, 0, 0], [0.5, 0, 0], [0, 0.5, 0]], np.float32); tri = np.array([[0, 1, 2]], np.uint32)
    om = oracle_mod.OracleMesh(tri_pos, tri); mm = api.MeshMap(tri_pos, tri)
    ed = om.edge_distances(); mm.setCosts(np.zeros(3, np.float32), ed)
    sfs, sps = _goals(tri_pos, tri, [0, 0])
    sps[1] = [0.1, 0.1, 0.0]
    got = api.CVPMeshPlanner(mm).waveFrontPropagationBatchFields(sfs, sps)
    assert got["outcome"] == 0 and (got["pred"] == np.arange(3)).all() and (got["cutting_face"] == 0).all()
    _check_oracle(om, ed, np.zeros(3, np.float32), sfs, sps, got)
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_counts(api, oracle_mod):
    """one and three goals (clusters of CTAs per wavefront); more goals than wavefronts in flight"""
    rng = np.random.default_rng(3)
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 40, costs=(rng.random(1600) * 0.8), factor=1.0)
    pl = api.CVPMeshPlanner(mm)
    sfs, sps = _goals(pos, faces, rng.choice(om.F, 3, replace=False))
    for n in (1, 3):
        got = pl.waveFrontPropagationBatchFields(sfs[:n], sps[:n])
        assert got["outcome"] == 0
        _check_oracle(om, w, vc, sfs[:n], sps[:n], got)
        _check_single(pl, sfs[:n], sps[:n], got)
    mm.close()
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 20, costs=(rng.random(400) * 0.8), factor=1.0)
    sfs, sps = _goals(pos, faces, rng.integers(0, om.F, 600))
    got = api.CVPMeshPlanner(mm).waveFrontPropagationBatchFields(sfs, sps)
    assert got["outcome"] == 0
    ref = {}
    for k, f in enumerate(sfs):
        if int(f) not in ref:
            ref[int(f)] = om.cvp(w, vc, int(f), sps[k])
        r = ref[int(f)]
        assert _same(got["dist"][k], r["dist"]) and (got["pred"][k] == r["pred"]).all(), k
        assert (got["cutting_face"][k] == r["cutting_face"]).all() and _direction_ok(got["direction"][k], r["direction"]), k
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_output_modes(api, oracle_mod):
    """each output alone and all four together, in host mode and with device pointers: the same bytes"""
    rng = np.random.default_rng(8)
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 30, costs=(rng.random(900) * 0.8), factor=1.0)
    sfs, sps = _goals(pos, faces, rng.choice(om.F, 5, replace=False))
    rc, full = _raw(mm, sfs, sps)
    assert rc == 0
    _check_oracle(om, w, vc, sfs, sps, full)
    for key in KEYS:
        rc, one = _raw(mm, sfs, sps, want=(key,))
        assert rc == 0 and _same(one[key], full[key]), key
        assert all(one[k] is None for k in KEYS if k != key)
    # dist only through the public wrapper is the same as mnb_cvp_batch's rows
    assert _same(api.CVPMeshPlanner(mm).waveFrontPropagationBatch(sfs, sps)["dist"], full["dist"])
    # decided by the loaded library: the CPU interpreter (it exports its fiber switch) cannot dereference device pointers
    on_gpu = not hasattr(mm.L, "mnb_emu_switch")
    if on_gpu:
        import torch
        mk = lambda dt: torch.full((sfs.size, om.V), 7, dtype=dt, device="cuda")
        bufs = dict(dist=mk(torch.float32), pred=mk(torch.int32), direction=mk(torch.float32), cutting_face=mk(torch.int32))
        ptr = lambda t: t.data_ptr(); back = lambda t: t.cpu().numpy(); fill = lambda t: t.fill_(7)
    else:
        bufs = dict(dist=np.full((sfs.size, om.V), 7, np.float32), pred=np.full((sfs.size, om.V), 7, np.uint32),
                    direction=np.full((sfs.size, om.V), 7, np.float32), cutting_face=np.full((sfs.size, om.V), 7, np.int32))
        ptr = lambda a: a.ctypes.data; back = lambda a: a

        def fill(a):
            a[:] = 7
    sync = (lambda: torch.cuda.synchronize()) if on_gpu else (lambda: None)
    mm.use_device_pointers(True)
    try:
        assert mm.cvp_batch_fields_dev(sfs, sps, 1.0, *[ptr(bufs[k]) for k in KEYS]) == 0
        sync()
        for key in KEYS:
            assert _same(back(bufs[key]), full[key]), key
        for key in KEYS:
            for b in bufs.values():
                fill(b)
            args = [ptr(bufs[k]) if k == key else 0 for k in KEYS]
            assert mm.cvp_batch_fields_dev(sfs, sps, 1.0, *args) == 0
            sync()
            assert _same(back(bufs[key]), full[key]), key
            assert all((back(bufs[k]).view(np.uint32) == np.full(1, 7, bufs_dtype(k)).view(np.uint32)).all() for k in KEYS if k != key)
    finally:
        mm.use_device_pointers(False)
    mm.close()


def bufs_dtype(key):
    return {"dist": np.float32, "pred": np.uint32, "direction": np.float32, "cutting_face": np.int32}[key]


@pytest.mark.gpu
def test_cvp_batch_fields_arguments_and_state(api, oracle_mod):
    """no costs installed -> MNB_E_STATE (-3); n == 0, NULL seeds and all outputs NULL -> MNB_E_ARG (-1); a seed face >= F
    -> INVALID_START (52) with nothing written"""
    pos, faces = mesh_case(20, True)
    mm = api.MeshMap(pos, faces)
    sfs, sps = _goals(pos, faces, [3, 4])
    rc, _ = _raw(mm, sfs, sps)
    assert rc == -3
    om = oracle_mod.OracleMesh(pos, faces); ed = om.edge_distances(); mm.setCosts(np.zeros(om.V, np.float32), ed)
    bad = np.array([3, om.F, 4], np.uint32); bsp = np.zeros((3, 3), np.float32)
    rc, out = _raw(mm, bad, bsp)
    assert rc == 52 and all((out[k].view(np.uint32) == np.full(1, 7, bufs_dtype(k)).view(np.uint32)).all() for k in KEYS)
    rc, _ = _raw(mm, sfs, sps, want=())
    assert rc == -1
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    dist = np.empty((2, om.V), np.float32)
    assert mm.L.mnb_cvp_batch_fields(mm._ctx, 0, p(sfs), p(sps), 1.0, p(dist), None, None, None) == -1
    assert mm.L.mnb_cvp_batch_fields(mm._ctx, 2, None, p(sps), 1.0, p(dist), None, None, None) == -1
    assert mm.L.mnb_cvp_batch_fields(mm._ctx, 2, p(sfs), None, 1.0, p(dist), None, None, None) == -1
    with pytest.raises(ValueError):
        api.CVPMeshPlanner(mm).waveFrontPropagationBatchFields(sfs, sps, want=("dist", "vectors"))
    rc, out = _raw(mm, sfs, sps)
    assert rc == 0
    _check_oracle(om, ed, np.zeros(om.V, np.float32), sfs, sps, out)
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_after_other_calls(api, oracle_mod):
    """the last mnb_cvp's back-tracking path and mnb_vector_map(pred = NULL) are unchanged by a batch; rows follow
    mnb_update_vertex_costs; single plans after the batch stay exact"""
    rng = np.random.default_rng(21)
    costs = (0.45 + 0.45 * np.sin(3.0 * mesh_case(50, True)[0][:, 0])).astype(np.float32)
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 50, costs=costs, factor=1.0)
    pl = api.CVPMeshPlanner(mm)
    sfs, sps = _goals(pos, faces, rng.choice(om.F, 6, replace=False))
    _check_oracle(om, w, vc, sfs, sps, pl.waveFrontPropagationBatchFields(sfs, sps))
    changed = np.unique(rng.choice(om.V, 200, replace=False)).astype(np.uint32)
    mm.layerChanged(changed, (rng.random(changed.size) * 0.9).astype(np.float32), 1.0)
    vc2, w2 = mm.costs()
    assert (w2 != w).any()
    _check_oracle(om, w2, vc2, sfs, sps, pl.waveFrontPropagationBatchFields(sfs, sps))
    sv, sf, sp = centre_seed(pos, faces, (0.2, 0.25))
    rv, rf, rp = centre_seed(pos, faces, (0.8, 0.7))
    out = np.empty((om.V, 3), np.float32)
    vec = lambda: (mm.L.mnb_vector_map(mm._ctx, None, None, None, out.ctypes.data_as(C.c_void_p)), out.copy())[1]
    c0 = pl.waveFrontPropagation(sf, sp, rf)
    assert c0["outcome"] == 0
    bt0 = pl.backtrack(rp, rf); vm0 = vec()
    pl.waveFrontPropagation(sf, sp, rf)
    for want in (KEYS, ("dist",)):               # host staging of every output, and the potentials-only kernel
        assert pl.waveFrontPropagationBatchFields(sfs, sps, want=want)["outcome"] == 0
        bt1 = pl.backtrack(rp, rf); vm1 = vec()
        assert bt0["outcome"] == bt1["outcome"] == 0 and len(bt0["positions"]) > 5
        assert _same(bt0["positions"], bt1["positions"]) and (bt0["faces"] == bt1["faces"]).all()
        assert _same(vm0, vm1)
    # single plans after the batch
    one = pl.waveFrontPropagation(int(sfs[0]), sps[0])
    ref = om.cvp(w2, vc2, int(sfs[0]), sps[0])
    assert _same(one["dist"], ref["dist"]) and (one["pred"] == ref["pred"]).all() and (one["cutting_face"] == ref["cutting_face"]).all()
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_rows_feed_vector_map(api, oracle_mod):
    """rows k of pred / direction / cutting face are a CVPMeshPlanner::computeVectorMap input (cvp:204-239): the vector map
    of row k equals that of the single plan for goal k"""
    rng = np.random.default_rng(4)
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 50, costs=(rng.random(2500) * 0.8).astype(np.float32), factor=1.0)
    pl = api.CVPMeshPlanner(mm)
    sfs, sps = _goals(pos, faces, [centre_seed(pos, faces, uv)[1] for uv in ((0.3, 0.3), (0.7, 0.4), (0.5, 0.8))])
    got = pl.waveFrontPropagationBatchFields(sfs, sps)
    for k in range(len(sfs)):
        vm = pl.computeVectorMap(got["pred"][k], got["direction"][k], got["cutting_face"][k])
        one = pl.waveFrontPropagation(int(sfs[k]), sps[k])
        ref = pl.computeVectorMap(one["pred"], one["direction"], one["cutting_face"])
        assert (np.isnan(vm) == np.isnan(ref)).all() and (vm[~np.isnan(ref)].view(np.uint32) == ref[~np.isnan(ref)].view(np.uint32)).all()
        assert np.isfinite(vm).any()
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_cancel(api, oracle_mod):
    """mnb_cancel from another thread during a batch -> CANCELED (51); the persistent groups take no new goals, and the
    next call succeeds"""
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 60)
    mm.set_tuning(0.005, 1, 0)         # narrow band: many rounds per wavefront
    pl = api.CVPMeshPlanner(mm)
    rng = np.random.default_rng(2)
    n = 8
    while True:                        # grow the batch until it takes long enough for the cancel to land inside it
        sfs, sps = _goals(pos, faces, rng.integers(0, om.F, n))
        t0 = time.perf_counter(); full = pl.waveFrontPropagationBatchFields(sfs, sps, want=("pred",)); t_full = time.perf_counter() - t0
        assert full["outcome"] == 0
        if t_full > 0.2 or n >= 16384:
            break
        n *= 4
    assert t_full > 0.05, t_full
    outcomes = []

    def run():
        t1 = time.perf_counter(); o = pl.waveFrontPropagationBatchFields(sfs, sps, want=("pred",))["outcome"]
        outcomes.append((o, time.perf_counter() - t1))
    t = threading.Thread(target=run)
    t.start(); time.sleep(0.25 * t_full); mm.cancel(); t.join()
    assert outcomes[0][0] == 51, outcomes
    assert outcomes[0][1] < 0.85 * t_full, (outcomes, t_full)
    got = pl.waveFrontPropagationBatchFields(sfs[:2], sps[:2])
    assert got["outcome"] == 0
    _check_oracle(om, w, vc, sfs[:2], sps[:2], got)
    mm.close()


@pytest.mark.gpu
def test_cvp_batch_fields_large_mesh(api, oracle_mod):
    """1 M-vertex terrain, 64 goals, 4 rows against the oracle"""
    from mesh_navigation_b200 import synth
    pos, faces, om, mm, vc, w = _map(api, oracle_mod, 1000)
    gv = synth.batch_goal_vertices(om.V, 64, seed=1234)
    gi, gj = np.minimum(gv % 1000, 998), np.minimum(gv // 1000, 998)    # the grid face at each goal vertex
    sfs, sps = _goals(pos, faces, 2 * (gj * 999 + gi))
    got = api.CVPMeshPlanner(mm).waveFrontPropagationBatchFields(sfs, sps)
    assert got["outcome"] == 0 and np.isfinite(got["dist"]).all()
    _check_oracle(om, w, vc, sfs, sps, got, rows=[0, 21, 42, 63])
    mm.close()


def test_cvp_batch_fields_on_the_cpu_interpreter():
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
