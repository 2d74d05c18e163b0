"""Multi-GPU entry points of the C ABI (mnb_group_*, mnb_cvp_batch_sharded; include/meshnav_b200.h): one process, N devices,
goal k on rank k mod N, fields all-gathered by NCCL inside the library.  Runs with every device count the box offers (a
single device exercises the sharding / layout code without NCCL)."""
import ctypes as C

import numpy as np
import pytest

from tests.util import mesh_case

pytestmark = pytest.mark.gpu


def test_sharded_batch_through_the_c_abi(oracle_mod):
    import torch
    from mesh_navigation_b200 import _lib, api
    L = _lib.load()
    ndev = max(1, min(2, torch.cuda.device_count()))
    pos, faces = mesh_case(90, True)
    om = oracle_mod.OracleMesh(pos, faces)
    ed = om.edge_distances(); vc = np.zeros(om.V, np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for f in ("mnb_group_create", "mnb_group_set_mesh", "mnb_group_set_costs", "mnb_cvp_batch_sharded", "mnb_group_read_fields"):
        getattr(L, f).restype = C.c_int32
    L.mnb_group_row.restype = C.c_uint32; L.mnb_group_size.restype = C.c_int32
    L.mnb_group_last_error.restype = C.c_char_p
    L.mnb_cvp_batch_sharded.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_double, C.c_int32]
    L.mnb_group_read_fields.argtypes = [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32, C.c_void_p]
    L.mnb_group_set_mesh.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    L.mnb_group_set_costs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.mnb_group_row.argtypes = [C.c_void_p, C.c_uint32]; L.mnb_group_size.argtypes = [C.c_void_p]; L.mnb_group_destroy.argtypes = [C.c_void_p]
    devs = (C.c_int32 * ndev)(*range(ndev)); grp = C.c_void_p()
    assert L.mnb_group_create(ndev, devs, C.byref(grp)) == 0 and L.mnb_group_size(grp) == ndev
    assert L.mnb_cvp_batch_sharded(grp, 1, p(np.zeros(1, np.uint32)), p(np.zeros(3, np.float32)), 1.0, 1) == -3      # MNB_E_STATE: no map yet
    edges = np.ascontiguousarray(om.edges, np.uint32)
    assert L.mnb_group_set_mesh(grp, om.V, om.F, p(pos), p(faces), p(edges), edges.shape[0]) == 0
    assert L.mnb_group_set_costs(grp, p(vc), p(ed), None) == 0
    rng = np.random.default_rng(3)
    n = 7                                                                  # ragged: ranks own 4 and 3 goals
    sfs = rng.integers(0, om.F, n).astype(np.uint32); sps = np.stack([pos[faces[f]].mean(0) for f in sfs]).astype(np.float32)
    rc = L.mnb_cvp_batch_sharded(grp, n, p(sfs), p(sps), 1.0, 1)
    assert rc == 0, L.mnb_group_last_error(grp)
    pad = (n + ndev - 1) // ndev
    assert [L.mnb_group_row(grp, k) for k in range(n)] == [(k % ndev) * pad + k // ndev for k in range(n)]
    for rank in range(ndev):                                               # every device holds every field after the gather
        out = np.empty((n, om.V), np.float32)
        assert L.mnb_group_read_fields(grp, rank, 0, n, p(out)) == 0
        for k in range(n):
            ref = om.cvp(ed, vc, int(sfs[k]), sps[k])["dist"]
            assert (out[k].view(np.uint32) == ref.view(np.uint32)).all(), (rank, k)
    # dynamic obstacles: the change set goes to every replica (mnb_group_update_vertex_costs), the next sharded batch plans on it
    L.mnb_group_update_vertex_costs.restype = C.c_int32
    L.mnb_group_update_vertex_costs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_double]
    ch = rng.choice(om.V, om.V // 6, replace=False).astype(np.uint32)
    nv = (rng.random(ch.size) * 0.9).astype(np.float32)
    assert L.mnb_group_update_vertex_costs(grp, ch.size, p(ch), p(nv), 0, 0.0, 1.5) == 0
    vc2 = vc.copy(); vc2[ch] = nv
    w2 = ed.copy(); om.update_edge_weights(vc2, ed, 1.5, ch, w2)
    assert L.mnb_cvp_batch_sharded(grp, n, p(sfs), p(sps), 1.0, 1) == 0, L.mnb_group_last_error(grp)
    for rank in range(ndev):
        out = np.empty((n, om.V), np.float32)
        assert L.mnb_group_read_fields(grp, rank, 0, n, p(out)) == 0
        for k in range(n):
            ref = om.cvp(w2, vc2, int(sfs[k]), sps[k])["dist"]
            assert (out[k].view(np.uint32) == ref.view(np.uint32)).all(), ("after update", rank, k)
    L.mnb_group_destroy(grp)
