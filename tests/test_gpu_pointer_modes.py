"""Pointer modes of the C ABI: every array-taking entry point that no other test file calls with device pointers runs on
two contexts with the same history, one in host-pointer mode (MNB_PTR_HOST) and one in device-pointer mode
(MNB_PTR_DEVICE), and the two must agree bit for bit: every output array (as uint32 words, bytes for uint8 arrays), the
return code and every count.  Outputs start filled with a sentinel, so elements a call must not write (past a returned
count, or a NULL output's share of the staging) keep it in both modes.  The batch, matrix, field-repair and
inflation-repair calls have pointer-mode tests of their own.  The GPU tests run with -m gpu on an H100; the last test
replays them on the CPU interpreter of the kernels (tests/emu)."""
import ctypes as C
import mmap
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.util import centre_seed, disc_lethals, mesh_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


class Out:
    """an output array of n elements, filled with the sentinel"""

    def __init__(self, n, dtype=np.float32):
        self.n, self.dtype = n, np.dtype(dtype)

    def initial(self):
        return np.full(self.n * self.dtype.itemsize, SENTINEL, np.uint8).view(self.dtype)


class InOut:
    """an array the call reads and writes"""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a)

    def initial(self):
        return self.a.copy()


class Ptrs:
    """a host array of pointers to arrays in the pointer mode (the layers of the combination updates); None stays NULL"""

    def __init__(self, arrays):
        self.arrays = arrays


class Count:
    """a uint32 the call writes through a host pointer"""


def _bits(a):
    a = np.ascontiguousarray(a).reshape(-1)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(np.uint32)


class Twin:
    """two contexts on one map: [0] in host-pointer mode, [1] in device-pointer mode.  Device arrays are torch CUDA
    tensors on an H100 and plain host arrays on the CPU interpreter of the kernels, decided by the loaded library (the
    interpreter exports its fiber switch)."""

    def __init__(self, api, pos, faces):
        self.maps = [api.MeshMap(pos, faces), api.MeshMap(pos, faces)]
        self.maps[1].use_device_pointers(True)
        self.V, self.F, self.E = self.maps[0].V, self.maps[0].F, self.maps[0].E
        self.on_gpu = not hasattr(self.maps[0].L, "mnb_emu_switch")
        self.keep = []         # device arrays outlive their call: mnb_cvp_backtrack reads the last plan's rows

    def close(self):
        for m in self.maps:
            m.close()

    def _device(self, a):
        """a device copy of a and a function that reads it back"""
        a = np.ascontiguousarray(a)
        if self.on_gpu:
            import torch
            t = torch.from_numpy(a.reshape(-1).view(np.uint8).copy()).cuda()
            self.keep.append(t)
            return t.data_ptr(), lambda: t.cpu().numpy().view(a.dtype).reshape(a.shape)
        # the interpreter runs a cooperative or cluster launch as one forked process per CTA: what such a kernel writes
        # reaches the caller's memory only when that memory is shared
        d = np.frombuffer(mmap.mmap(-1, max(a.nbytes, 1)), np.uint8, a.nbytes).view(a.dtype).reshape(a.shape)
        d[...] = a
        self.keep.append(d)
        return d.ctypes.data, lambda: d.copy()

    def _run(self, mode, fn, args):
        reads, cargs = [], []

        def array(a):
            if mode == 0:
                a = np.ascontiguousarray(a)
                self.keep.append(a)
                return a.ctypes.data, lambda: a
            return self._device(a)

        for x in args:
            if isinstance(x, (Out, InOut)):
                p, back = array(x.initial())
                reads.append(back); cargs.append(C.c_void_p(p))
            elif isinstance(x, np.ndarray):
                cargs.append(C.c_void_p(array(x)[0]))
            elif isinstance(x, Ptrs):
                ptrs = (C.c_void_p * len(x.arrays))(*[None if a is None else array(a)[0] for a in x.arrays])
                self.keep.append(ptrs); cargs.append(C.cast(ptrs, C.c_void_p))
            elif isinstance(x, Count):
                c = C.c_uint32(0xA5A5A5A5)
                reads.append(lambda c=c: c.value); cargs.append(C.byref(c))
            else:
                cargs.append(x)
        m = self.maps[mode]
        rc = getattr(m.L, fn)(m._ctx, *cargs)
        if mode == 1 and self.on_gpu:
            import torch
            torch.cuda.synchronize()
        return [rc] + [r() for r in reads]

    def call(self, fn, *args):
        """fn(ctx, *args) on both contexts; asserts that they agree and returns [rc, outputs and counts in argument order]
        of the host-pointer one.  Arguments: numpy arrays are inputs in the pointer mode, Out / InOut / Ptrs / Count as
        above, anything else (scalars, NULL, host-only arrays as c_void_p, byref structs) is passed as it is."""
        host, dev = self._run(0, fn, args), self._run(1, fn, args)
        assert len(host) == len(dev)
        for k, (h, d) in enumerate(zip(host, dev)):
            if isinstance(h, np.ndarray):
                assert h.shape == d.shape and (_bits(h) == _bits(d)).all(), f"{fn}: output {k} differs between the pointer modes"
            else:
                assert h == d, f"{fn}: {'return code' if k == 0 else f'count {k}'} {h} (host) != {d} (device)"
        return host


def _host(a):
    """an array that is a host pointer in either mode (seed and robot positions, combination defaults and weights)"""
    return np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def _twin(api, n=20, seed=3):
    rng = np.random.default_rng(seed)
    pos, faces = mesh_case(n, True)
    tw = Twin(api, pos, faces)
    vc = (rng.random(tw.V) * 0.8).astype(np.float32)
    ed = tw.maps[0].edgeDistances()
    w = tw.call("mnb_compute_edge_weights", vc, 1.0, Out(tw.E))[1]
    assert np.isfinite(w).all() and (w >= ed).all()
    return tw, rng, pos, faces, vc, w


def _tail_kept(a, n):
    return (a.reshape(-1).view(np.uint8)[n * a.dtype.itemsize:] == SENTINEL).all()


@pytest.mark.gpu
def test_costs_pointer_modes(api):
    """mnb_compute_edge_weights, mnb_set_costs with and without the invalid mask, mnb_get_costs, mnb_update_vertex_costs
    with costs indexed by position and by vertex"""
    tw, rng, pos, faces, vc, w = _twin(api)
    V, E = tw.V, tw.E
    rc, w0 = tw.call("mnb_compute_edge_weights", vc, 0.0, Out(E))
    assert rc == 0 and not (w0 == w).all()
    assert tw.call("mnb_compute_edge_weights", vc, 2.0, None) == [0]
    assert tw.call("mnb_set_costs", vc, w, None) == [0]
    rc, gc, gw = tw.call("mnb_get_costs", Out(V), Out(E))
    assert rc == 0 and (_bits(gc) == _bits(vc)).all() and (_bits(gw) == _bits(w)).all()
    invalid = (rng.random(V) < 0.05).astype(np.uint8)
    assert tw.call("mnb_set_costs", vc, w, invalid) == [0]
    assert tw.call("mnb_get_costs", None, Out(E))[1].shape == (E,)
    changed = rng.choice(V, 40, replace=False).astype(np.uint32)
    costs_n = (rng.random(40) * 0.9).astype(np.float32)
    costs_n[::7] = np.inf
    assert tw.call("mnb_update_vertex_costs", changed.size, changed, costs_n, 0, 0.0, 1.0) == [0]
    rc, gc, gw = tw.call("mnb_get_costs", Out(V), Out(E))
    assert (_bits(gc[changed]) == _bits(costs_n)).all() and not (gw == w).all()
    costs_v = (rng.random(V) * 0.5).astype(np.float32)
    changed2 = rng.choice(V, 25, replace=False).astype(np.uint32)
    assert tw.call("mnb_update_vertex_costs", changed2.size, changed2, costs_v, 1, 0.25, 1.0) == [0]
    assert tw.call("mnb_update_vertex_costs", changed2.size, changed2, costs_v, 1, 0.25, 0.0) == [0]
    rc, gc, gw = tw.call("mnb_get_costs", Out(V), Out(E))
    assert (_bits(gc[changed2]) == _bits(costs_v[changed2])).all()
    tw.close()


@pytest.mark.gpu
@pytest.mark.parametrize("average", [False, True])
def test_combination_updates_pointer_modes(api, average):
    """mnb_max_combination_update / mnb_avg_combination_update with and without lethal masks"""
    tw, rng, pos, faces, vc, w = _twin(api)
    V = tw.V
    layers = [(rng.random(V) * 2.0).astype(np.float32) for _ in range(3)]
    layers[1][::5] = np.nan                             # no entry: the layer's default
    lethal = [(rng.random(V) < 0.1).astype(np.uint8), None, (rng.random(V) < 0.05).astype(np.uint8)]
    defaults = np.float32([0.1, 0.5, 0.0])
    weights = np.float32([0.5, 1.5, 1.0])
    changed = np.unique(rng.choice(V, 120)).astype(np.uint32)
    io_costs = (rng.random(V) * 3.0).astype(np.float32)
    io_lethal = (rng.random(V) < 0.02).astype(np.uint8)
    fn = "mnb_avg_combination_update" if average else "mnb_max_combination_update"
    head = (_host(weights),) if average else ()
    for ll, il in ((Ptrs(lethal), InOut(io_lethal)), (None, None), (Ptrs([None, None, lethal[2]]), InOut(io_lethal))):
        res = tw.call(fn, 3, Ptrs(layers), _host(defaults), *head, ll, changed.size, changed, InOut(io_costs), il)
        assert res[0] == 0 and not (_bits(res[1]) == _bits(io_costs)).all()
        if il is not None:
            assert res[2].any()
    tw.close()


@pytest.mark.gpu
def test_layers_locate_vector_map_pointer_modes(api):
    """mnb_compute_layers with and without clearance, mnb_locate, mnb_vector_map on given rows and (pred = NULL) on the
    last plan's"""
    from mesh_navigation_b200 import _lib
    tw, rng, pos, faces, vc, w = _twin(api)
    V = tw.V
    P = _lib.LayerParams.defaults()
    rc, costs, comb, mask = tw.call("mnb_compute_layers", C.byref(P), None, Out(6 * V), Out(V), Out(V, np.uint8))
    assert rc == 0 and np.isfinite(comb).any()
    clearance = (rng.random(V) * 1.5).astype(np.float32)
    clearance[::9] = np.inf
    rc, costs2, comb2, mask2 = tw.call("mnb_compute_layers", C.byref(P), clearance, Out(6 * V), Out(V), Out(V, np.uint8))
    assert rc == 0 and not (_bits(costs2) == _bits(costs)).all() and mask2.any()
    assert tw.call("mnb_compute_layers", C.byref(P), clearance, None, Out(V), None)[0] == 0
    pts = (pos[rng.choice(V, 50)] + rng.normal(size=(50, 3)) * 0.03).astype(np.float32)
    pts[-1] = [1e3, 1e3, 1e3]                            # far off the mesh: no containing face
    rc, nv, fc, ba = tw.call("mnb_locate", 50, pts, Out(50, np.uint32), Out(50, np.int32), Out(150))
    assert rc == 0 and (nv < V).all() and (fc >= 0).sum() > 25 and fc[-1] == -1
    assert tw.call("mnb_locate", 50, pts, None, Out(50, np.int32), None)[0] == 0
    assert tw.call("mnb_set_costs", vc, w, None) == [0]
    sv, sf, sp = centre_seed(pos, faces, (0.3, 0.3))
    rc, dist, pred, dirs, cut = tw.call("mnb_cvp", sf, _host(sp), -1, 10.0, 0.0, Out(V), Out(V, np.uint32), Out(V), Out(V, np.int32))
    assert rc == 0 and np.isfinite(dist).sum() > V // 2
    rc, vm = tw.call("mnb_vector_map", pred, dirs, cut, Out(3 * V))
    assert rc == 0 and (vm != 0).any()
    rc, vm_pred = tw.call("mnb_vector_map", pred, None, None, Out(3 * V))
    assert rc == 0 and not (_bits(vm_pred) == _bits(vm)).all()
    rc, vm_last = tw.call("mnb_vector_map", None, None, None, Out(3 * V))
    assert rc == 0 and (_bits(vm_last) == _bits(vm)).all()
    tw.close()


@pytest.mark.gpu
def test_single_plans_pointer_modes(api):
    """mnb_cvp with every output, with only out_dist and with out_dist NULL; mnb_cvp_backtrack after each (in device mode
    it reads the caller's rows or the scratch); mnb_dijkstra with and without a robot vertex, seed == robot, NULL rows"""
    tw, rng, pos, faces, vc, w = _twin(api)
    V = tw.V
    assert tw.call("mnb_set_costs", vc, w, None) == [0]
    sv, sf, sp = centre_seed(pos, faces, (0.3, 0.3))
    rv, rf, rp = centre_seed(pos, faces, (0.75, 0.65))
    cvp = lambda *outs: tw.call("mnb_cvp", sf, _host(sp), rf, 10.0, 0.3, *outs)
    bt = lambda max_points=4096, faces_out=True: tw.call("mnb_cvp_backtrack", _host(rp), rf, 0.1, max_points, Out(3 * max_points),
                                                        Out(max_points, np.uint32) if faces_out else None, Count())
    rc, dist, pred, dirs, cut = cvp(Out(V), Out(V, np.uint32), Out(V), Out(V, np.int32))
    assert rc == 0 and np.isfinite(dist).sum() > V // 2
    ref = bt()
    assert ref[0] == 0 and 5 < ref[3] < 4096 and _tail_kept(ref[1], 3 * ref[3]) and _tail_kept(ref[2], ref[3])
    short = bt(max_points=4)
    assert 0 < short[3] <= 4 and (_bits(short[1][:3 * short[3]]) == _bits(ref[1][:3 * short[3]])).all()
    assert cvp(Out(V), None, None, None)[0] == 0
    assert (_bits(bt(faces_out=False)[1]) == _bits(ref[1])).all()
    rc, pred2, dirs2, cut2 = cvp(None, Out(V, np.uint32), Out(V), Out(V, np.int32))
    assert rc == 0 and (pred2 == pred).all() and (_bits(dirs2) == _bits(dirs)).all() and (cut2 == cut).all()
    assert (_bits(bt()[1]) == _bits(ref[1])).all()
    assert tw.call("mnb_cvp", sf, _host(sp), -1, 0.05, 0.0, Out(V), None, Out(V), None)[0] == 0
    # Dijkstra
    rc, dd, dp = tw.call("mnb_dijkstra", sv, rv, 10.0, 0.3, Out(V), Out(V, np.uint32))
    assert rc == 0 and np.isfinite(dd).sum() > V // 2 and dp[rv] != rv
    assert tw.call("mnb_dijkstra", sv, -1, 10.0, 0.0, Out(V), Out(V, np.uint32))[0] == 0
    rc, dd2 = tw.call("mnb_dijkstra", sv, rv, 10.0, 0.3, Out(V), None)
    assert rc == 0 and (_bits(dd2) == _bits(dd)).all()
    rc, dp2 = tw.call("mnb_dijkstra", sv, rv, 10.0, 0.3, None, Out(V, np.uint32))
    assert rc == 0 and (dp2 == dp).all()
    rc, dd3, dp3 = tw.call("mnb_dijkstra", sv, sv, 10.0, 0.3, Out(V), Out(V, np.uint32))
    assert rc == 0 and dd3[sv] == 0 and (dp3 == np.arange(V)).all()
    assert tw.call("mnb_dijkstra", sv, sv, 10.0, 0.3, None, None) == [0]
    tw.close()


@pytest.mark.gpu
def test_inflation_pointer_modes(api):
    """mnb_inflate with and without the invalid mask and with NULL outputs, mnb_inflation_update (elements past the count
    keep the sentinel), mnb_inflation_vector_map, mnb_inflation_vector_at"""
    from mesh_navigation_b200 import _lib
    tw, rng, pos, faces, vc, w = _twin(api)
    V, F = tw.V, tw.F
    params = _lib.InflationParams(0.2, 0.5, 1.0, 0.99, 1.0)
    lethals = np.ascontiguousarray(disc_lethals(pos, 3, 0.15, seed=5), np.uint32)
    invalid = (rng.random(V) < 0.03).astype(np.uint8)
    rc, dist, cost = tw.call("mnb_inflate", lethals, lethals.size, None, C.byref(params), Out(V), Out(V))
    assert rc == 0 and np.isfinite(dist).sum() > 2 * lethals.size
    assert tw.call("mnb_inflate", lethals, lethals.size, invalid, C.byref(params), None, Out(V))[0] == 0
    assert tw.call("mnb_inflate", lethals, lethals.size, invalid, C.byref(params), Out(V), None)[0] == 0
    rc, vec = tw.call("mnb_inflation_vector_map", Out(3 * V))
    assert rc == 0 and (vec != 0).any()
    fq = rng.choice(F, 30).astype(np.uint32)
    bary = rng.dirichlet(np.ones(3), 30).astype(np.float32)
    rc, va = tw.call("mnb_inflation_vector_at", 30, fq, bary, Out(90))
    assert rc == 0 and (va != 0).any()
    moved = np.ascontiguousarray(disc_lethals(pos, 3, 0.15, seed=6), np.uint32)
    rc, d2, c2, chg, n = tw.call("mnb_inflation_update", moved, moved.size, invalid, C.byref(params), Out(V), Out(V),
                                 Out(V, np.uint32), Count())
    assert rc == 0 and 0 < n < V and _tail_kept(chg, n)
    rc, chg2, n2 = tw.call("mnb_inflation_update", lethals, lethals.size, None, C.byref(params), None, None, Out(V, np.uint32), Count())
    assert rc == 0 and 0 < n2 < V and _tail_kept(chg2, n2)
    assert tw.call("mnb_inflation_update", lethals, lethals.size, None, C.byref(params), None, None, None, Count())[0] == 0
    rc, vec2 = tw.call("mnb_inflation_vector_map", Out(3 * V))
    assert rc == 0 and (vec2 != 0).any()
    tw.close()


@pytest.mark.gpu
def test_rays_pointer_modes(api):
    """mnb_cast_rays with per-ray and shared directions and NULL outputs, mnb_obstacle_update (lethal and changed lists
    past their counts keep the sentinel; with and without the cost map), mnb_normal_clearance with and without normals"""
    from mesh_navigation_b200 import _lib
    tw, rng, pos, faces, vc, w = _twin(api)
    V = tw.V
    n = 64
    origins = (pos[rng.choice(V, n)] + np.float32([0, 0, 0.5])).astype(np.float32)
    dirs = rng.normal(size=(n, 3)).astype(np.float32)
    dirs[:, 2] = -np.abs(dirs[:, 2]) - 0.5
    res = tw.call("mnb_cast_rays", n, origins, dirs, 3, Out(n, np.uint8), Out(n), Out(n, np.uint32), Out(3 * n))
    assert res[0] == 0 and 0 < res[1].sum() < n
    down = np.float32([0, 0, -1])
    res = tw.call("mnb_cast_rays", n, origins, down, 0, Out(n, np.uint8), None, Out(n, np.uint32), None)
    assert res[0] == 0 and res[1].all()
    assert tw.call("mnb_cast_rays", n, origins, dirs, 3, None, Out(n), None, Out(3 * n))[0] == 0
    P = _lib.ObstacleParams(); P.max_obstacle_dist = 10.0; P.robot_height = 0.4
    P.tf[:] = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]; P.down_axis[:] = [0.0, 0.0, -1.0]
    assert tw.call("mnb_obstacle_reset") == [0]
    for step in range(3):
        pts = pos[rng.choice(V, 200)] + np.float32([0, 0, 0.2])
        pts[::3, 2] += 1.0                                # above the robot: no obstacle
        costs = Out(V) if step != 1 else None
        res = tw.call("mnb_obstacle_update", pts.shape[0], pts.astype(np.float32), C.byref(P), Out(V, np.uint32), Count(),
                      Out(V, np.uint32), Count(), costs)
        rc, le, nl, ch, nc = res[:5]
        assert rc == 0 and 0 < nl < V and 0 < nc < V and _tail_kept(le, nl) and _tail_kept(ch, nc)
    res = tw.call("mnb_obstacle_update", 0, None, C.byref(P), None, Count(), Out(V, np.uint32), Count(), Out(V))
    assert res[0] == 0 and res[1] == 0 and res[3] > 0
    vn = tw.maps[0].vertexNormals()
    rc, cl = tw.call("mnb_normal_clearance", vn, Out(V))
    assert rc == 0
    rc, cl0 = tw.call("mnb_normal_clearance", None, Out(V))
    assert rc == 0 and (_bits(cl0) == _bits(cl)).all()
    vn2 = vn.copy(); vn2[:, 2] *= -1.0
    assert tw.call("mnb_normal_clearance", vn2, Out(V))[0] == 0
    tw.close()


def test_pointer_modes_on_the_cpu_interpreter():
    """the GPU tests above with the kernels compiled by g++ against tests/emu, on 4 emulated SMs"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    env = dict(os.environ, MNB_EMU_SMS="4")
    r = subprocess.run([sys.executable, runner, os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, tail
