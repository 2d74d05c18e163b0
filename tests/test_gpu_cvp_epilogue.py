"""The single-plan CVP epilogue (predecessors, directions and cutting faces of mnb_cvp and mnb_cvp_replan) in both of its
replays: k_cvp_epilogue replays a vertex in registers from its ELL row when it has at most 8 faces and every source label
is a plain one-level time, and hands every other vertex to the CSR replay of k_cvp_epilogue_csr.  mnb_debug_set_cvp_epilogue
(ctx, 1) hands every replayed vertex to the CSR replay, so that each case runs both replays on the same wave.

Every case checks
  * the oracle (CVPMeshPlanner::waveFrontPropagation): potentials, predecessors and cutting faces bit for bit and the same
    outcome; directions bit for bit on the CPU interpreter of the kernels, and on the GPU at most one float ulp apart on
    fewer than 1e-4 of the vertices (CUDA's and glibc's double acos may differ in the last bit);
  * the row replay against the CSR replay: all four outputs bit for bit;
  * the routing: the hand-off count (mnb_debug_get_epilogue_csr) equals the vertices the rule selects, computed here from
    the labels (mnb_debug_get_labels) and the faces -- reached, eligible, not a seed, and more than 8 faces or a face
    neighbour whose label word carries cascade levels (z | w != 0); with every vertex handed off, all reached eligible
    non-seeds;
  * the deep_labels statistic (counted in the epilogue) against the labels' ext words;
  * mnb_cvp (robot face -1) against the row of mnb_cvp_batch_fields, whose epilogue runs the CSR replay in line.
Each case family asserts that it reaches the vertices it is there for.  The GPU tests run with -m gpu on an H100; the last
test replays them on the CPU interpreter of the kernels (tests/emu)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from mesh_navigation_b200 import synth
from tests.util import centre_seed, mesh_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUTS = ("dist", "pred", "direction", "cutting_face")
FUZZ = ("deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour")
INF_BITS = 0x7F800000
EXT_POOL = 0x80000000
ROW_FACES = 8                     # ELL_W: the faces an ELL row holds
WHEELS = (3, 7, 8, 9, 12, 13, 24)  # face counts of the hub vertices of wheel_mesh; 12 / 13: replay() / replay_big()


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


def _ulps(a, b):
    """distance in float ulps (sign-magnitude bits mapped onto a monotonic integer line)"""
    def line(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(line(a) - line(b))


def wheel_mesh(ks=WHEELS, n_points=2000, extent=4.0, seed=7):
    """Delaunay mesh of random points with a hub vertex for each k in ks, ringed by k points in a cleared disc: hub i has
    exactly ks[i] faces.  Returns pos, faces and the hub vertex ids."""
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(seed)
    xy = rng.random((n_points, 2)) * extent
    centres = np.array([[0.7 + 0.9 * (i % 4), 1.2 + 1.6 * (i // 4)] for i in range(len(ks))]) * (extent / 4.0)
    keep = np.ones(len(xy), bool)
    for c in centres:
        keep &= np.linalg.norm(xy - c, axis=1) > 0.5
    parts, hubs, n = [xy[keep]], [], int(keep.sum())
    for c, k in zip(centres, ks):
        ang = np.linspace(0, 2 * np.pi, k, endpoint=False) + rng.random() * 0.3
        parts.append(c + 0.2 * np.stack([np.cos(ang), np.sin(ang)], 1) * (1 + 0.002 * rng.random(k))[:, None])
        parts.append(c[None, :])
        n += k
        hubs.append(n)
        n += 1
    xy = np.concatenate(parts)
    faces = Delaunay(xy).simplices.astype(np.uint32)
    a, b, c3 = xy[faces[:, 0]], xy[faces[:, 1]], xy[faces[:, 2]]
    area = (b[:, 0] - a[:, 0]) * (c3[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c3[:, 0] - a[:, 0])
    faces[area < 0] = faces[area < 0][:, [0, 2, 1]]
    faces = faces[np.abs(area) > 1e-9]
    z = 0.4 * np.sin(xy[:, 0] * 1.3) * np.cos(xy[:, 1] * 0.9)
    pos = np.concatenate([xy, z[:, None]], 1).astype(np.float32)
    hubs = np.array(hubs)
    assert (np.bincount(faces.reshape(-1), minlength=len(xy))[hubs] == np.array(ks)).all()
    return pos, faces, hubs


def _fuzz(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", f"fuzz_{name}.npz"))
    inv = d["inv"] if d["inv"].size else None
    return d["pos"], d["faces"], d["vc"], d["w"], inv, int(d["sf"]), d["sp"], int(d["rf"]), float(d["cl"])


def _face_with(faces, v, avoid=()):
    """a face that has vertex v and none of `avoid`"""
    for f in np.where((faces == v).any(1))[0]:
        if not np.isin(faces[f], avoid).any():
            return int(f)
    raise AssertionError(f"no face at vertex {v}")


class Map:
    """one mesh with its costs on one context; plan() runs a single plan in one epilogue mode and collects what the checks
    read (outputs, hand-off count, labels)"""

    def __init__(self, api, oracle_mod, pos, faces, vc=None, w=None, factor=1.0, invalid=None, cost_limit=1.0,
                 goal_dist_offset=0.3):
        self.api, self.pos, self.faces = api, pos, np.asarray(faces, np.uint32)
        self.om = None if oracle_mod is None else oracle_mod.OracleMesh(pos, faces)     # None: no oracle (w is given)
        self.mm = api.MeshMap(pos, faces)
        self.V = self.mm.V
        self.vc = np.zeros(self.V, np.float32) if vc is None else np.asarray(vc, np.float32)
        self.w = self.om.edge_weights(self.vc, self.om.edge_distances(), factor) if w is None else w
        self.invalid = invalid
        self.mm.setCosts(self.vc, self.w, invalid)
        self.pl = api.CVPMeshPlanner(self.mm, cost_limit=cost_limit, goal_dist_offset=goal_dist_offset)
        self.nfaces = np.bincount(self.faces.reshape(-1), minlength=self.V)
        self.exact = hasattr(self.mm.L, "mnb_emu_switch")     # the CPU interpreter: its acos is the oracle's
        self.cluster = -1                                      # single plans on k_cvp_grid (mnb_set_tuning's default)

    def close(self):
        self.mm.close()

    def mode(self, m):
        assert self.mm.L.mnb_debug_set_cvp_epilogue(self.mm._ctx, m) == 0

    def handed_off(self):
        n = C.c_uint32(0xFFFFFFFF)
        assert self.mm.L.mnb_debug_get_epilogue_csr(self.mm._ctx, C.byref(n)) == 0
        return int(n.value)

    def labels(self):
        lab = np.empty((self.V, 4), np.uint32); root = np.empty(self.V, np.uint32); ext = np.empty(self.V, np.uint32)
        L, ctx = self.mm.L, self.mm._ctx
        assert L.mnb_debug_get_labels(ctx, lab.ctypes.data) == 0
        assert L.mnb_debug_get_label_sides(ctx, root.ctypes.data, ext.ctypes.data, None, 0) == 0
        return lab, ext

    def tune(self, cluster):
        self.mm.set_tuning(0.0, cluster, 0)
        self.cluster = cluster

    def plan(self, sf, sp, rf=-1, mode=0, replan=None):
        """mnb_cvp (replan None) or mnb_cvp_replan with the changed vertices `replan`, in epilogue mode `mode`"""
        self.mode(mode)
        # The interpreter runs the CTAs of the cooperative k_cvp_grid as processes, and that launch stalls now and then
        # there when a robot face arms the goal cutoff (so did the parent build's); it runs those plans on k_cvp<1>.
        one_cta = self.exact and rf >= 0 and self.cluster == -1
        if one_cta:
            self.mm.set_tuning(0.0, 1, 0)
        try:
            if replan is None:
                r = self.pl.waveFrontPropagation(sf, sp, rf)
            else:
                r = self.pl.waveFrontReplan(sf, sp, rf, replan)
            r["epi_csr"] = self.handed_off()
            if replan is None:
                r["labels"], r["ext"] = self.labels()
        finally:
            self.mode(0)
            if one_cta:
                self.mm.set_tuning(0.0, -1, 0)
        return r

    def eligible(self):
        el = ~(self.vc.astype(np.float64) >= self.pl.cost_limit)
        return el if self.invalid is None else el & (self.invalid == 0)

    def routing(self, lab, sf):
        """the vertices the row replay hands to the CSR replay, by the rule of CvpProblem::replay_row"""
        reached = lab[:, 0] != INF_BITS
        seed = np.zeros(self.V, bool); seed[self.faces[sf]] = True
        replayed = reached & self.eligible() & ~seed
        cascade = (lab[:, 2] | lab[:, 3]) != 0
        nb = np.zeros(self.V, bool)
        for k in range(3):
            np.logical_or.at(nb, self.faces[:, k], cascade[self.faces[:, (k + 1) % 3]] | cascade[self.faces[:, (k + 2) % 3]])
        big = self.nfaces > ROW_FACES
        return dict(replayed=replayed, big=replayed & big, cascade_row=replayed & ~big & nb, plain_row=replayed & ~big & ~nb,
                    handoff=replayed & (big | nb))

    def oracle(self, sf, sp, rf=-1, vc=None, w=None):
        return self.om.cvp(self.w if w is None else w, self.vc if vc is None else vc, sf, sp, rf, invalid=self.invalid,
                           cost_limit=self.pl.cost_limit, goal_dist_offset=self.pl.goal_dist_offset)

    def check_oracle(self, got, ref, what=""):
        """the comparison with the oracle; returns the number of directions that are not bit-identical"""
        assert got["outcome"] == ref["outcome"], (what, got["outcome"], ref["outcome"])
        for k in ("dist", "pred", "cutting_face"):
            assert _same(got[k], ref[k]), f"{what} {k}: {np.count_nonzero(got[k].view(np.uint32) != ref[k].view(np.uint32))} differ"
        u = _ulps(got["direction"], ref["direction"])
        if self.exact:
            assert (u == 0).all(), f"{what} direction: {np.count_nonzero(u)} differ"
        else:
            assert u.max() <= 1 and np.count_nonzero(u) < 1e-4 * u.size, f"{what} direction: {np.count_nonzero(u)} differ, max {u.max()} ulp"
        return int(np.count_nonzero(u))

    def check(self, sf, sp, rf=-1, what="", batch=True):
        """every check of the module docstring on one plan; returns the routing sets and both runs"""
        ref = self.oracle(sf, sp, rf)
        row = self.plan(sf, sp, rf, 0)
        csr = self.plan(sf, sp, rf, 1)
        n_dir = self.check_oracle(row, ref, what)
        for k in OUTS:
            assert _same(row[k], csr[k]), f"{what} row vs CSR replay: {k}"
        assert _same(row["labels"], csr["labels"])                         # the same wave
        rt = self.routing(row["labels"], sf)
        assert row["epi_csr"] == rt["handoff"].sum(), (what, row["epi_csr"], int(rt["handoff"].sum()))
        assert csr["epi_csr"] == rt["replayed"].sum(), (what, csr["epi_csr"], int(rt["replayed"].sum()))
        lab, ext = row["labels"], row["ext"]
        deep = (lab[:, 0] != INF_BITS) & ((lab[:, 3] >> 31) != 0) & ((ext & EXT_POOL) != 0)
        assert row["deep_labels"] == csr["deep_labels"] == deep.sum(), (what, row["deep_labels"], int(deep.sum()))
        if batch and rf < 0:
            fields = self.pl.waveFrontPropagationBatchFields(np.array([sf], np.uint32), np.asarray(sp, np.float32)[None])
            assert fields["outcome"] == 0
            for k in OUTS:
                assert _same(fields[k][0], row[k]), f"{what} batch fields row vs mnb_cvp: {k}"
        print(f"[epilogue] {what}: replayed {int(rt['replayed'].sum())}, row {int(rt['replayed'].sum() - row['epi_csr'])}, "
              f"CSR {row['epi_csr']} (>8 faces {int(rt['big'].sum())}, cascade sources {int(rt['cascade_row'].sum())}), "
              f"deep labels {row['deep_labels']}; directions not bit-identical to the oracle's: {n_dir} of {self.V}")
        return rt, row, csr


def _shared_triggers(faces, lab):
    """per vertex: does it have two faces with both sources reached and the same later source (by plain pop time (a1, id))?
    Their face times tie, and the corner order decides which is replayed first"""
    V = lab.shape[0]
    fin = lab[:, 0] != INF_BITS
    a1 = lab[:, 1].view(np.float32)
    keys = []
    for k in range(3):
        c, v1, v2 = faces[:, k].astype(np.int64), faces[:, (k + 1) % 3].astype(np.int64), faces[:, (k + 2) % 3].astype(np.int64)
        later = np.where((a1[v1] > a1[v2]) | ((a1[v1] == a1[v2]) & (v1 > v2)), v1, v2)
        ok = fin[v1] & fin[v2]
        keys.append(c[ok] * V + later[ok])
    u, n = np.unique(np.concatenate(keys), return_counts=True)
    out = np.zeros(V, bool)
    out[u[n >= 2] // V] = True
    return out


def _wheels(api, oracle_mod, seed=7, factor=1.0, costs="random"):
    pos, faces, hubs = wheel_mesh(seed=seed)
    rng = np.random.default_rng(seed)
    vc = (rng.random(pos.shape[0]) * 0.6).astype(np.float32) if costs == "random" else np.zeros(pos.shape[0], np.float32)
    return Map(api, oracle_mod, pos, faces, vc, factor=factor), hubs


@pytest.mark.gpu
@pytest.mark.parametrize("factor", [0.0, 1.0])
def test_epilogue_face_counts(api, oracle_mod, factor):
    """reached, eligible non-seed vertices with exactly 3..8 faces (the row replay), 9 (the first one past the row), 12 and
    13 (replay() / replay_big()) and 24 faces"""
    cs, hubs = _wheels(api, oracle_mod, factor=factor)
    try:
        _, sf, sp = centre_seed(cs.pos, cs.faces, (0.45, 0.5))
        rt, row, _ = cs.check(sf, sp, what=f"wheels factor {factor}")
        for k in (3, 4, 5, 6, 7, 8, 9, 12, 13, 24):
            assert (rt["replayed"] & (cs.nfaces == k)).any(), f"no replayed vertex with {k} faces"
        assert rt["replayed"][hubs].all()
        assert (rt["handoff"] & (cs.nfaces == 9)).any() and not (rt["handoff"] & (cs.nfaces == 8) & ~rt["cascade_row"]).any()
        # faces that fire: the hubs were updated through several of their faces
        assert (row["cutting_face"][hubs] >= 0).all()
    finally:
        cs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FUZZ + ("cost_walls",))
def test_epilogue_source_labels(api, oracle_mod, name):
    """labels with cascade levels: vertices with at most 8 faces and a cascade member among their face neighbours (handed
    off), and ones with plain sources only (replayed on the row)"""
    if name == "cost_walls":
        pos, faces = mesh_case(40, True)
        rng = np.random.default_rng(2)
        vc = (rng.random(pos.shape[0]) * 0.7).astype(np.float32)
        vc[(pos[:, 0] > 1.5) & (pos[:, 0] < 1.8) & (pos[:, 1] > 0.8)] = 0.95      # a costly wall with a gap
        cs = Map(api, oracle_mod, pos, faces, vc, factor=2.5)
        _, sf, sp = centre_seed(pos, faces, (0.3, 0.6))
    else:
        pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz(name)
        cs = Map(api, oracle_mod, pos, faces, vc, w, invalid=inv, cost_limit=cl)
    try:
        rt, row, _ = cs.check(sf, sp, what=name)
        assert rt["cascade_row"].any(), "no row-sized vertex with a cascade member among its sources"
        assert rt["plain_row"].any()
        if name.startswith("deep_cascade"):
            assert row["deep_labels"] > 0
    finally:
        cs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("costs", ["zero", "quantised"])
def test_epilogue_exact_ties(api, oracle_mod, costs):
    """unjittered planar grid: faces fired by the same trigger give equal candidates, and the corner order decides"""
    pos, faces = synth.grid_mesh(30, 30, jitter=0.0, terrain=False)
    rng = np.random.default_rng(4)
    vc = np.zeros(pos.shape[0], np.float32) if costs == "zero" else (np.floor(rng.random(pos.shape[0]) * 4) * 0.2).astype(np.float32)
    cs = Map(api, oracle_mod, pos, faces, vc, factor=0.0 if costs == "zero" else 1.0)
    try:
        for uv in ((0.5, 0.5), (0.2, 0.7)):
            _, sf, sp = centre_seed(pos, faces, uv)
            rt, row, _ = cs.check(sf, sp, what=f"ties {costs} {uv}")
            assert rt["plain_row"].sum() > 0.5 * rt["replayed"].sum()
            assert _shared_triggers(cs.faces, row["labels"])[rt["plain_row"]].sum() > 0.5 * rt["plain_row"].sum()
    finally:
        cs.close()


@pytest.mark.gpu
def test_epilogue_seeds(api, oracle_mod):
    """seed faces at a 9-face and an 8-face vertex, a seed over the cost limit, an invalid seed (neither expands), a seed
    point next to a vertex (very unequal seed potentials)"""
    pos, faces, hubs = wheel_mesh(seed=11)
    V = pos.shape[0]
    rng = np.random.default_rng(11)
    vc = (rng.random(V) * 0.6).astype(np.float32)
    nf = np.bincount(faces.reshape(-1), minlength=V)
    h9, h8 = int(hubs[list(WHEELS).index(9)]), int(hubs[list(WHEELS).index(8)])
    f_over = _face_with(faces, int(hubs[list(WHEELS).index(12)]))
    vc[faces[f_over][0]] = 1.5                                              # a seed over the cost limit
    invalid = np.zeros(V, np.uint8)
    f_inv = _face_with(faces, int(hubs[list(WHEELS).index(13)]))
    invalid[faces[f_inv][1]] = 1                                            # an invalid seed
    invalid[rng.choice(V, 10, replace=False)] = 1
    invalid[faces[[_face_with(faces, h9), _face_with(faces, h8)]].reshape(-1)] = 0
    cs = Map(api, oracle_mod, pos, faces, vc, invalid=invalid)
    try:
        for what, f in (("seed at 9 faces", _face_with(faces, h9)), ("seed at 8 faces", _face_with(faces, h8)),
                        ("seed over the limit", f_over), ("invalid seed", f_inv)):
            sp = pos[faces[f]].mean(0).astype(np.float32)
            rt, row, _ = cs.check(f, sp, what=what)
            s = faces[f]
            assert (row["pred"][s] == s).all() and (row["cutting_face"][s] == f).all()
            assert rt["replayed"].sum() > 0.5 * V
        assert nf[faces[_face_with(faces, h9)]].max() == 9 and nf[faces[_face_with(faces, h8)]].max() == 8
        # a seed point 1e-3 from one corner of the face of the 8-face hub: its seed potential is tiny next to the others'
        f = _face_with(faces, h8)
        sp = (0.998 * pos[h8] + 0.001 * pos[faces[f]].sum(0) - 0.001 * pos[h8]).astype(np.float32)
        d = np.linalg.norm(pos[faces[f]] - sp, axis=1)
        assert d.min() < 0.01 * d.max()
        cs.check(f, sp, what="seed point near a vertex")
    finally:
        cs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0.0, 0.3])
def test_epilogue_goal_cutoff(api, oracle_mod, offset):
    """a robot face: the goal cutoff filters the faces a vertex beyond it may fire (CvpProblem::expands); an unreachable
    robot (NO_PATH_FOUND, 54)"""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz("cutoff_cascade")
    cs = Map(api, oracle_mod, pos, faces, vc, w, invalid=inv, cost_limit=cl, goal_dist_offset=offset)
    try:
        rt, row, _ = cs.check(sf, sp, rf, what=f"cutoff offset {offset}")
        assert row["outcome"] == 0 and (~np.isfinite(row["dist"])).sum() > 0.1 * cs.V     # the cutoff left a part unreached
        assert rt["handoff"].any() and rt["plain_row"].any()
    finally:
        cs.close()
    # two components: the robot face lies in the one the wave cannot reach
    pos1, faces1 = mesh_case(20, True)
    pos = np.concatenate([pos1, pos1 + np.array([10.0, 0, 0], np.float32)])
    faces = np.concatenate([faces1, faces1 + len(pos1)]).astype(np.uint32)
    rng = np.random.default_rng(1)
    cs = Map(api, oracle_mod, pos, faces, (rng.random(len(pos)) * 0.6).astype(np.float32), goal_dist_offset=offset)
    try:
        _, sf, sp = centre_seed(pos1, faces1, (0.4, 0.4))
        rt, row, _ = cs.check(sf, sp, len(faces1) + 17, what=f"unreachable robot offset {offset}")
        assert row["outcome"] == 54
        assert np.isinf(row["dist"][len(pos1):]).all() and rt["replayed"].sum() > 0.5 * len(pos1)
    finally:
        cs.close()


@pytest.mark.gpu
def test_epilogue_unreached_and_ineligible(api, oracle_mod):
    """invalid vertices, costs at and over the cost limit, a +inf wall, a disconnected second component: no replay, and
    the in-line writes (self, 0, -1)"""
    pos1, faces1, _ = wheel_mesh(seed=5)
    n1 = len(pos1)
    pos = np.concatenate([pos1, pos1 + np.array([10.0, 0, 0], np.float32)])
    faces = np.concatenate([faces1, faces1 + n1]).astype(np.uint32)
    V = len(pos)
    rng = np.random.default_rng(5)
    vc = (rng.random(V) * 0.6).astype(np.float32)
    vc[rng.choice(V, 60, replace=False)] = 1.0                 # at the cost limit: not eligible
    vc[rng.choice(V, 60, replace=False)] = 3.0
    vc[(pos[:, 0] > 2.9) & (pos[:, 0] < 3.1)] = np.inf          # +inf: not eligible either
    invalid = (rng.random(V) < 0.03).astype(np.uint8)
    cs = Map(api, oracle_mod, pos, faces, vc, invalid=invalid)
    try:
        _, sf, sp = centre_seed(pos1, faces1, (0.3, 0.5))
        while not (cs.eligible()[faces[sf]]).all():
            sf += 1
        sp = pos[faces[sf]].mean(0).astype(np.float32)
        rt, row, _ = cs.check(sf, sp, what="unreached and ineligible")
        seed = np.zeros(V, bool); seed[faces[sf]] = True
        none = ~rt["replayed"] & ~seed
        assert (~cs.eligible() & (row["labels"][:, 0] == INF_BITS))[:n1].sum() > 100 and np.isinf(row["dist"][n1:]).all()
        assert (invalid[:n1] != 0).sum() > 10 and np.isinf(vc[:n1]).sum() > 10
        assert (row["pred"][none] == np.nonzero(none)[0]).all() and (row["cutting_face"][none] == -1).all()
        assert (row["direction"][none] == 0).all()
    finally:
        cs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [-1, 1, 2, 16])
def test_epilogue_launch_forms(api, oracle_mod, cluster):
    """k_cvp_grid (cluster -1) and k_cvp<CS>: the epilogue runs on the labels each leaves"""
    for name in ("deep_cascade_delaunay", "wheels"):
        if name == "wheels":
            cs, _ = _wheels(api, oracle_mod, seed=3)
            _, sf, sp = centre_seed(cs.pos, cs.faces, (0.6, 0.4))
        else:
            pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz(name)
            cs = Map(api, oracle_mod, pos, faces, vc, w, invalid=inv, cost_limit=cl)
        try:
            cs.tune(cluster)
            rt, _, _ = cs.check(sf, sp, what=f"{name} cluster {cluster}", batch=False)
            assert rt["handoff"].any() and rt["plain_row"].any()
        finally:
            cs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [-1, 2])
def test_epilogue_replan(api, oracle_mod, cluster):
    """mnb_cvp_replan resumed after a cost change: the epilogue runs on the resident workspace; both replays against the
    oracle, each other and a fresh plan"""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz("deep_cascade_delaunay")
    cs = Map(api, oracle_mod, pos, faces, vc, w, invalid=inv, cost_limit=cl)
    try:
        cs.tune(cluster)
        first = cs.plan(sf, sp, replan=np.empty(0, np.uint32))
        far = int(np.argmax(np.where(np.isfinite(first["dist"]), first["dist"], 0.0)))
        disc = np.where(np.linalg.norm(pos[:, :2] - pos[far, :2], axis=1) < 0.35)[0].astype(np.uint32)
        vals = (0.5 * vc[disc] + 0.3).astype(np.float32)
        cs.mm.layerChanged(disc, vals, 1.0)
        vc2, w2 = cs.mm.costs()
        cs.vc = vc2
        ref = cs.oracle(sf, sp, vc=vc2, w=w2)
        fresh = cs.plan(sf, sp)
        row = cs.plan(sf, sp, replan=disc, mode=0)
        assert 0 < row["settled"] < fresh["settled"], (row["settled"], fresh["settled"])
        cs.mm.layerChanged(disc, vals, 1.0)                          # the same values again: a resumed wave on equal costs
        csr = cs.plan(sf, sp, replan=disc, mode=1)
        assert 0 < csr["settled"] < fresh["settled"]
        for r, what in ((row, "replan row"), (csr, "replan CSR")):
            cs.check_oracle(r, ref, what)
            for k in OUTS:
                assert _same(r[k], fresh[k]), f"{what} vs fresh plan: {k}"
        seed = np.zeros(cs.V, bool); seed[faces[sf]] = True
        replayed = np.isfinite(csr["dist"]) & cs.eligible() & ~seed
        assert csr["epi_csr"] == replayed.sum() and 0 < row["epi_csr"] < csr["epi_csr"]
        print(f"[epilogue] replan cluster {cluster}: replayed {int(replayed.sum())}, CSR {row['epi_csr']}")
    finally:
        cs.close()


@pytest.mark.gpu
def test_epilogue_state_between_calls(api, oracle_mod):
    """a plan that hands off many vertices, then one that hands off few, in both orders: each count is the plan's own and
    no stale list entry is replayed; a host-mode call with one output alone writes the full call's values"""
    pos, faces, vc, w, inv, sf, sp, rf, cl = _fuzz("cutoff_cascade")
    cs = Map(api, oracle_mod, pos, faces, vc, w, invalid=inv, cost_limit=cl, goal_dist_offset=0.0)
    try:
        _, sf2, _ = centre_seed(pos, faces, (0.8, 0.3))
        while not cs.eligible()[faces[sf2]].all():
            sf2 += 1
        sp2 = pos[faces[sf2]].mean(0).astype(np.float32)
        _, rf2, _ = centre_seed(pos, faces, (0.85, 0.36))
        plans = {"many": (sf, sp, -1, 1), "few": (sf2, sp2, rf2, 0)}
        refs = {k: cs.oracle(*p[:3]) for k, p in plans.items()}
        counts = {}
        for order in (("many", "few"), ("few", "many")):
            for key in order:
                f, s, r, mode = plans[key]
                got = cs.plan(f, s, r, mode)
                cs.check_oracle(got, refs[key], key)
                rt = cs.routing(got["labels"], f)
                assert got["epi_csr"] == rt["replayed" if mode else "handoff"].sum(), (key, got["epi_csr"])
                counts[key] = got["epi_csr"]
        assert counts["many"] > 4 * counts["few"] > 0, counts
        # the seeds of "few" are in the list of "many", and its cutoff leaves vertices that "many" reached: a stale entry
        # replayed there would write a predecessor
        assert np.isfinite(refs["many"]["dist"][faces[sf2]]).all() and (np.isinf(refs["few"]["dist"]) & np.isfinite(refs["many"]["dist"])).any()
        # one output alone, in both modes
        L, ctx = cs.mm.L, cs.mm._ctx
        full = cs.plan(sf, sp)
        for mode in (0, 1):
            cs.mode(mode)
            try:
                for k, t in (("pred", np.uint32), ("direction", np.float32)):
                    out = np.full(cs.V, 7, t)
                    args = [out.ctypes.data_as(C.c_void_p) if kk == k else None for kk in OUTS]
                    rc = L.mnb_cvp(ctx, sf, np.ascontiguousarray(sp, np.float32).ctypes.data_as(C.c_void_p), -1, cl,
                                   cs.pl.goal_dist_offset, *args)
                    assert rc == 0 and _same(out, full[k]), (mode, k)
            finally:
                cs.mode(0)
    finally:
        cs.close()


@pytest.mark.gpu
def test_epilogue_large_terrain(api, oracle_mod):
    """1 M-vertex terrain with the layer stack's costs (fused layers Max-combined with the inflation of their lethals and
    obstacle discs; lethal walls, back-steps): the row replay against the CSR replay and the routing"""
    from mesh_navigation_b200.api import InflationLayer
    n = 1000
    pos, faces = mesh_case(n, True)
    mm = api.MeshMap(pos, faces)
    try:
        mm.setCosts(np.zeros(mm.V, np.float32), mm.edgeDistances())
        Ly = mm.computeLayers()
        le = np.union1d(np.where(Ly["lethal_mask"] != 0)[0], synth.disc_lethals_grid(pos, n, n, 200, 0.3)).astype(np.uint32)
        I = InflationLayer(mm).waveCostInflation(le)
        final = np.maximum(Ly["combined"], np.nan_to_num(I["cost"], nan=0.0)).astype(np.float32)
        w = mm.computeEdgeWeights(final, 1.0)
    finally:
        mm.close()
    cs = Map(api, None, pos, faces, final, w)
    try:
        free = np.where(final < 0.5)[0]
        v = int(free[np.argmin(np.linalg.norm(pos[free, :2] - pos[:, :2].mean(0), axis=1))])
        f = 2 * (min(v // n, n - 2) * (n - 1) + min(v % n, n - 2))
        while not (final[faces[f]] < 1.0).all():
            f += 1
        sp = pos[faces[f]].mean(0).astype(np.float32)
        row = cs.plan(f, sp, mode=0)
        csr = cs.plan(f, sp, mode=1)
        assert row["outcome"] == csr["outcome"] == 0
        for k in OUTS:
            assert _same(row[k], csr[k]), k
        rt = cs.routing(row["labels"], f)
        assert row["epi_csr"] == rt["handoff"].sum() and csr["epi_csr"] == rt["replayed"].sum()
        assert rt["replayed"].sum() > cs.V // 2 and (final >= 1.0).sum() > 1000 and rt["cascade_row"].any()
        print(f"[epilogue] 1M terrain: replayed {int(rt['replayed'].sum())}, CSR {row['epi_csr']} "
              f"(cascade sources {int(rt['cascade_row'].sum())}), deep labels {row['deep_labels']}")
    finally:
        cs.close()


def test_cvp_epilogue_on_the_cpu_interpreter():
    """the GPU tests above (minus the 1 M-vertex one) with the kernels compiled by g++ against tests/emu, on 4 emulated
    SMs, in the default warp order and in a randomised one"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    for extra in ({}, {"MNB_EMU_SHUFFLE": "3"}):
        env = dict(os.environ, MNB_EMU_SMS="4", **extra)
        r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider", "-k", "not large_terrain"],
                           cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
        tail = (r.stdout + r.stderr)[-3000:]
        assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"{extra}:\n{tail}"
