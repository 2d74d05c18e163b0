"""Vector-field back-tracking (mnb_cvp_backtrack / k_backtrack: cvp_mesh_planner.cpp:920-951 over MeshMap::meshAhead)
against the oracle's sequential walk on the same device vector map: outcome, point count, positions as uint32 and faces,
bit for bit.  The cases are where the warp-parallel face search could leave the sequential order: fine grids (one step's
search lists more faces than the shared-memory list holds), every step width, vertices of high degree (one listed face's
expansions outgrow their shared-memory row), the repulsive field, walks off the mesh border, the max_points limit and a
bad robot face.  The GPU tests run with -m gpu on an H100; the last test replays them on the CPU interpreter of the
kernels (tests/emu)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from mesh_navigation_b200 import synth
from tests.util import centre_seed, disc_lethals

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_STATE, NO_PATH, INVALID_GOAL = -3, 54, 53


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _grid(h, extent, terrain):
    """an n x n grid of spacing h (cut by the diagonal (0,0)-(1,1) of every cell); terrain: gentle hills"""
    n = int(round(extent / h)) + 1
    return synth.grid_mesh(n, n, h=h, terrain=terrain, z_scale=0.3, wavelength=2.0)


def _costs(pos):
    lo, hi = pos[:, :2].min(0), pos[:, :2].max(0)
    u = (pos[:, :2] - lo) / (hi - lo)
    return (0.45 + 0.45 * np.sin(6.0 * u[:, 0]) * np.cos(4.0 * u[:, 1])).astype(np.float32)


def hub_mesh(degree, n_points=900, seed=3, extent=6.0):
    """Delaunay mesh of random points with a hub vertex (the last) in the middle, joined to a ring of `degree` vertices
    on one circle (so every ring vertex is the hub's neighbour); each ring vertex has 3 or 4 faces"""
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(seed)
    xy = rng.random((n_points, 2)) * extent
    c = np.array([extent * 0.5, extent * 0.5])
    xy = xy[np.linalg.norm(xy - c, axis=1) > 0.30]
    ang = (np.arange(degree) + 0.3 * rng.random(degree)) * (2 * np.pi / degree)
    xy = np.concatenate([xy, c + 0.22 * np.stack([np.cos(ang), np.sin(ang)], 1), c[None, :]])
    faces = Delaunay(xy).simplices.astype(np.uint32)
    a, b, c3 = xy[faces[:, 0]], xy[faces[:, 1]], xy[faces[:, 2]]
    area = (b[:, 0] - a[:, 0]) * (c3[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c3[:, 0] - a[:, 0])
    faces[area < 0] = faces[area < 0][:, [0, 2, 1]]
    faces = faces[np.abs(area) > 1e-9]
    z = 0.4 * np.sin(xy[:, 0] * 1.3) * np.cos(xy[:, 1] * 0.9)
    return np.concatenate([xy, z[:, None]], 1).astype(np.float32), faces


def _face_at(pos, faces, xy):
    """a face that contains the point xy (in the plane), and its centroid"""
    a, b, c = (pos[faces[:, k], :2].astype(np.float64) for k in range(3))
    p = np.asarray(xy, np.float64)
    cr = lambda u, v, w: (v[:, 0] - u[:, 0]) * (w[:, 1] - u[:, 1]) - (v[:, 1] - u[:, 1]) * (w[:, 0] - u[:, 0])
    pp = np.broadcast_to(p, a.shape)
    s = np.stack([cr(a, b, pp), cr(b, c, pp), cr(c, a, pp)], 1)
    f = int(np.where((s >= 0).all(1) | (s <= 0).all(1))[0][0])
    return f, pos[faces[f]].mean(0).astype(np.float32)


def _gpu_walk(mm, rp, rf, step, max_points):
    """mnb_cvp_backtrack through the C ABI (the error codes are not raised): (rc, positions, faces, error text)"""
    rp = np.ascontiguousarray(rp, np.float32)
    pos = np.empty((max_points, 3), np.float32); face = np.empty(max_points, np.uint32); n = C.c_uint32(0)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    rc = mm.L.mnb_cvp_backtrack(mm._ctx, p(rp), int(rf) & 0xffffffff, float(step), int(max_points), p(pos), p(face), C.byref(n))
    err = mm.L.mnb_last_error(mm._ctx).decode() if rc < 0 else ""
    return rc, pos[:n.value].copy(), face[:n.value].copy(), err


class Walks:
    """one map and one plan on the device; walk() runs mnb_cvp_backtrack and the oracle's walk on the device's vector
    map and asserts that they agree bit for bit"""

    def __init__(self, api, oracle_mod, pos, faces, weighted=True):
        self.api, self.pos, self.faces = api, pos, faces
        self.om = oracle_mod.OracleMesh(pos, faces)
        self.mm = api.MeshMap(pos, faces)
        self.vc = _costs(pos) if weighted else np.zeros(pos.shape[0], np.float32)
        self.mm.setCosts(self.vc, self.om.edge_weights(self.vc, self.om.edge_distances(), 1.0 if weighted else 0.0))
        self.pl = api.CVPMeshPlanner(self.mm)

    def plan(self, sf, sp, rf=-1):
        g = self.pl.waveFrontPropagation(sf, sp, rf)
        assert g["outcome"] == 0
        self.sf, self.sp = int(sf), np.asarray(sp, np.float32)
        self.vm = self.pl.computeVectorMap(g["pred"], g["direction"], g["cutting_face"])
        return g

    def oracle_walk(self, rp, rf, step=0.4, max_points=1 << 16, repulsive=None):
        rc, pp, pf = self.om.cvp_backtrack(self.vm, self.sp, self.sf, rp, rf, step, max_points, repulsive=repulsive)
        return (E_STATE if rc == -1 else rc), pp, pf

    def walk(self, rp, rf, step=0.4, max_points=1 << 16, repulsive=None):
        rc, pp, pf, err = _gpu_walk(self.mm, rp, rf, step, max_points)
        orc, opp, opf = self.oracle_walk(rp, rf, step, max_points, repulsive)
        assert rc == orc, (rc, orc, err)
        assert pp.shape == opp.shape, (pp.shape, opp.shape)
        bad = np.where((pp.view(np.uint32) != opp.view(np.uint32)).any(1))[0]
        assert bad.size == 0, f"{bad.size} of {len(pp)} points differ, the first at {bad[0]}: {pp[bad[0]]} vs {opp[bad[0]]}"
        assert (pf == opf).all()
        return rc, pp, pf, err


def _success(w, rp, rf, step=0.4, min_points=4):
    rc, pp, pf, _ = w.walk(rp, rf, step)
    assert rc == 0 and len(pp) >= min_points, (rc, len(pp))
    assert (pp[0] == rp).all() and (pp[-1] == w.sp).all() and pf[0] == rf and pf[-1] == w.sf
    return pp


# ---- resolution ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["along", "across"])
@pytest.mark.parametrize("kind", ["planar", "terrain"])
@pytest.mark.parametrize("h", [0.1, 0.05, 0.02, 0.012, 0.01, 0.007])
def test_backtrack_resolution(api, oracle_mod, h, kind, direction):
    """grids of 1.6 m at 10 cm down to 7 mm (at 1 cm one 0.4 m step lists ~5000 faces); paths along and across the
    diagonal that cuts the cells; the terrain with weighted costs, so the field curves"""
    pos, faces = _grid(h, 1.6, kind == "terrain")
    w = Walks(api, oracle_mod, pos, faces, weighted=kind == "terrain")
    s, r = ((0.12, 0.12), (0.88, 0.88)) if direction == "along" else ((0.12, 0.88), (0.88, 0.12))
    _, sf, sp = centre_seed(pos, faces, s)
    _, rf, rp = centre_seed(pos, faces, r)
    w.plan(sf, sp, rf)
    _success(w, rp, rf)
    w.mm.close()


# ---- step width ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("step", [0.05, 0.1, 0.4, 1.0, 2.5])
def test_backtrack_step_width(api, oracle_mod, step):
    """the walk ends on distance^2 <= step_width (cvp:925, as written): the map grows with the step so that every
    walk takes several steps; at 2.5 m on a 5 cm grid one step lists ~15000 faces.  The grid is flat: a straight
    step of metres leaves a hilly surface by more than the 0.4 m the face search accepts"""
    pos, faces = _grid(0.05, 2.0 + 2.4 * step, False)
    w = Walks(api, oracle_mod, pos, faces)
    _, sf, sp = centre_seed(pos, faces, (0.3, 0.35))
    _, rf, rp = centre_seed(pos, faces, (0.9, 0.85))
    w.plan(sf, sp, rf)
    _success(w, rp, rf, step)
    w.mm.close()


# ---- vertex degree -------------------------------------------------------------------------------------------------
def _hub_case(api, oracle_mod, degree, permuted):
    pos, faces = hub_mesh(degree)
    hub = pos.shape[0] - 1
    cnt = np.bincount(faces.ravel(), minlength=pos.shape[0])
    assert cnt[hub] == degree
    hub_faces = np.where((faces == hub).any(1))[0]
    sums = cnt[faces[hub_faces]].sum(1)
    if permuted:
        rng = np.random.default_rng(degree)
        pv = rng.permutation(pos.shape[0]); inv = np.empty_like(pv); inv[pv] = np.arange(pv.size)
        pf = rng.permutation(faces.shape[0]); finv = np.empty_like(pf); finv[pf] = np.arange(pf.size)
        pos, faces = np.ascontiguousarray(pos[pv]), np.ascontiguousarray(inv[faces].astype(np.uint32)[pf])
        hub_faces = finv[hub_faces]
    return pos, faces, hub_faces, sums


@pytest.mark.gpu
@pytest.mark.parametrize("permuted", [False, True])
@pytest.mark.parametrize("role", ["path", "robot"])
@pytest.mark.parametrize("degree", [24, 55, 60, 64, 65, 90, 200])
def test_backtrack_hub(api, oracle_mod, degree, role, permuted):
    """a hub vertex of high degree in the middle of a Delaunay mesh: on the path (the walk crosses it), or the robot
    face is one of its faces (the first search expands it first); the same with random vertex and face ids"""
    pos, faces, hub_faces, _ = _hub_case(api, oracle_mod, degree, permuted)
    w = Walks(api, oracle_mod, pos, faces)
    c = np.array([3.0, 3.0])
    sf, sp = _face_at(pos, faces, c + [-1.6, -1.1])
    if role == "path":
        rf, rp = _face_at(pos, faces, c + [1.5, 1.2])
    else:
        rf = int(hub_faces[0]); rp = pos[faces[rf]].mean(0).astype(np.float32)
    w.plan(sf, sp, rf)
    _success(w, rp, rf)
    w.mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("permuted", [False, True])
@pytest.mark.parametrize("total", [63, 64, 65])
def test_backtrack_expansion_row_edge(api, oracle_mod, total, permuted):
    """the robot face is a face of a degree-55 hub whose three vertices have `total` faces together: the first
    search expands it into exactly that many candidates (64 fill a shared-memory row, 65 do not fit)"""
    pos, faces, hub_faces, sums = _hub_case(api, oracle_mod, 55, permuted)
    assert (sums == total).any(), sorted(set(sums.tolist()))
    w = Walks(api, oracle_mod, pos, faces)
    rf = int(hub_faces[np.where(sums == total)[0][0]])
    assert np.bincount(faces.ravel(), minlength=pos.shape[0])[faces[rf]].sum() == total
    rp = pos[faces[rf]].mean(0).astype(np.float32)
    for s in ([-1.6, -1.1], [1.4, -1.5], [0.2, 1.8]):                  # three directions out of the face
        sf, sp = _face_at(pos, faces, np.array([3.0, 3.0]) + s)
        w.plan(sf, sp, rf)
        _success(w, rp, rf)
    w.mm.close()


# ---- repulsive field -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("h", [0.05, 0.01])
def test_backtrack_repulsive_field_exact(api, oracle_mod, h):
    """setRepulsiveField(True) on a disc-obstacle map: the oracle walks with the device's inflation distances and
    vector field, so the bent path is bit-exact"""
    pos, faces = _grid(h, 2.0, True)
    w = Walks(api, oracle_mod, pos, faces, weighted=False)
    infl = api.InflationLayer(w.mm)
    lethals = disc_lethals(pos, 6, 0.12, seed=12)
    dist = infl.waveCostInflation(lethals)["dist"]
    vec = infl.vectorMap()
    _, sf, sp = centre_seed(pos, faces, (0.1, 0.15))
    _, rf, rp = centre_seed(pos, faces, (0.9, 0.85))
    w.plan(sf, sp, rf)
    plain = _success(w, rp, rf)
    infl.setRepulsiveField(True)
    rc, bent, _, _ = w.walk(rp, rf, repulsive=dict(dist=dist, vectors=vec))
    infl.setRepulsiveField(False)
    assert rc in (0, NO_PATH)
    k = min(len(plain), len(bent))
    assert np.abs(plain[:k] - bent[:k]).max() > 1e-3, "the repulsive field left the path unchanged"
    w.mm.close()


# ---- search exhausted ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("h", [0.1, 0.01])
def test_backtrack_walks_off_the_border(api, oracle_mod, h):
    """robots near the border of a weighted terrain whose field the walk follows off the mesh: every face search
    lists all faces in reach (on the 1 cm grid more than 5000) and finds none -- NO_PATH_FOUND on both sides; and a
    robot position beyond the border, whose first search finds nothing"""
    pos, faces = _grid(h, 2.0, True)
    w = Walks(api, oracle_mod, pos, faces)
    _, sf, sp = centre_seed(pos, faces, (0.5, 0.04))
    w.plan(sf, sp)
    found = 0
    for fy in (0.97, 0.9, 0.5):
        for fx in np.linspace(0.05, 0.95, 19):
            _, rf, rp = centre_seed(pos, faces, (fx, fy))
            orc, opp, _ = w.oracle_walk(rp, rf)
            if orc == NO_PATH and len(opp) >= 2 and found < 3:
                assert w.walk(rp, rf)[0] == NO_PATH
                found += 1
    assert found > 0
    _, rf, rp = centre_seed(pos, faces, (0.5, 1.0))
    rp = rp + np.float32([0.0, 0.3, 0.0])
    rc, pp, _, _ = w.walk(rp, rf)
    assert rc == NO_PATH and len(pp) == 1
    w.mm.close()


# ---- max_points ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("h", [0.05, 0.01])
def test_backtrack_max_points(api, oracle_mod, h):
    """the smallest max_points that succeeds returns the oracle's path; one less is MNB_E_STATE, and the error
    text names max_points and nothing else"""
    pos, faces = _grid(h, 1.6, True)
    w = Walks(api, oracle_mod, pos, faces)
    _, sf, sp = centre_seed(pos, faces, (0.1, 0.1))
    _, rf, rp = centre_seed(pos, faces, (0.9, 0.9))
    w.plan(sf, sp, rf)
    full = _success(w, rp, rf, 0.1)
    n = len(full)
    rc, pp, _, _ = w.walk(rp, rf, 0.1, max_points=n)
    assert rc == 0 and (pp.view(np.uint32) == full.view(np.uint32)).all()
    rc, pp, _, err = w.walk(rp, rf, 0.1, max_points=n - 1)
    assert rc == E_STATE and len(pp) == n - 2 and (pp.view(np.uint32) == full[:n - 2].view(np.uint32)).all()
    assert "max_points" in err and "search" not in err, err
    w.mm.close()


# ---- whole plan ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_make_plan_fine_map(api, oracle_mod):
    """makePlan (wave seeded at the goal, then the walk from the robot) on a 1 cm map: its positions are the oracle's
    walk on the same field"""
    pos, faces = _grid(0.01, 1.6, True)
    w = Walks(api, oracle_mod, pos, faces)
    _, gf, gp = centre_seed(pos, faces, (0.8, 0.25))
    _, sf, sp = centre_seed(pos, faces, (0.15, 0.85))
    r = w.pl.makePlan(sp, sf, gp, gf)
    assert r["outcome"] == 0 and len(r["positions"]) >= 4
    w.plan(gf, gp, sf)
    orc, opp, opf = w.oracle_walk(sp, sf)
    assert orc == 0 and (opp.view(np.uint32) == r["positions"].view(np.uint32)).all() and (opf == r["faces"]).all()
    w.mm.close()


# ---- arguments -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_backtrack_robot_face_out_of_range(api, oracle_mod):
    """a robot face >= F (or -1) is MNB_INVALID_GOAL on both sides, with no points"""
    pos, faces = _grid(0.1, 1.6, False)
    w = Walks(api, oracle_mod, pos, faces)
    _, sf, sp = centre_seed(pos, faces, (0.2, 0.2))
    w.plan(sf, sp)
    rp = pos[faces[3]].mean(0)
    for rf in (faces.shape[0], faces.shape[0] + 7, -1):
        rc, pp, pf, _ = _gpu_walk(w.mm, rp, rf, 0.4, 64)
        orc, opp, opf = w.oracle_walk(rp, rf)
        assert rc == orc == INVALID_GOAL and len(pp) == len(opp) == 0
    w.mm.close()


def test_oracle_backtrack_face_arguments(oracle_mod):
    """the oracle walk checks its face arguments instead of reading past the face array"""
    pos, faces = _grid(0.1, 1.0, False)
    om = oracle_mod.OracleMesh(pos, faces)
    vm = np.zeros((om.V, 3), np.float32)
    p = pos[faces[0]].mean(0)
    assert om.cvp_backtrack(vm, p, 0, p, -1)[0] == INVALID_GOAL
    assert om.cvp_backtrack(vm, p, 0, p, om.F)[0] == INVALID_GOAL
    assert om.cvp_backtrack(vm, p, om.F, p, 0)[0] == 52
    assert om.cvp_backtrack(vm, p, 0, p, 0)[0] == 0


@pytest.mark.parametrize("shuffle, expr", [
    (None, "not nothing"),
    ("3", "(resolution and 0.01 and terrain) or (hub and 90) or expansion_row_edge or walks_off or max_points"),
])
def test_backtrack_on_the_cpu_interpreter(shuffle, expr):
    """the GPU tests above with the kernels compiled by g++ against tests/emu, on 4 emulated SMs, in the default warp
    order; a subset again in a randomised one"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    env = dict(os.environ, MNB_EMU_SMS="4", **({"MNB_EMU_SHUFFLE": shuffle} if shuffle else {}))
    r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider", "-k", expr],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=560)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"shuffle {shuffle}:\n{tail}"
