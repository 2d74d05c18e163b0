"""The single-plan wavefront kernels at every launch configuration the C ABI accepts, and past their shared-memory capacities.

k_cvp_grid, k_dijkstra_grid, k_cvp<CS>, k_dijkstra<CS> and k_inflate are run with every block size of mnb_set_tuning (128, 256,
512), every cluster size, in-round sweep counts from 0 to 64 (odd ones included) and band widths from half a dependency hop to
wider than the mesh.  Every run is compared with the oracle (potentials and distances bit for bit, predecessors and cutting
faces exactly, CVP directions within 1e-5) and with the default configuration's run of the same plan on the GPU, all outputs
bit for bit: the launch configuration may change the order of the work, never the result.

The capacity tests size their meshes from the SM count so that the round engine's per-CTA limits (Stage::SW_CAP sweep
slots and main-pass chunks, Stage::CAP staged entries) are exceeded, and prove it from the plan statistics."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests.util import centre_seed, delaunay_mesh, face_of_vertex, mesh_case

pytestmark = pytest.mark.gpu

FUZZ = ("deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour")
PLANS = FUZZ + ("noncausal_terrain", "delaunay_hub")
FULL = "deep_cascade_planar"                 # the fixture that runs every threads x sweeps x band combination
THREADS = (128, 256, 512)
CVP_SWEEPS = (0, 1, 2, 3, 11, 12, 64, -1)
DIJKSTRA_SWEEPS = (0, 1, 3, 15, 64, -1)
CLUSTERS = (1, 2, 4, 8, 16)
BANDS = ("half_hop", "default", "odd", "wide")
SW_CAP, STAGE_CAP = 1024, 3072               # Stage::SW_CAP and Stage::CAP (band_engine.cuh)


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _debug(mm, name, value):
    f = getattr(mm.L, name)
    f.argtypes = [C.c_void_p, C.c_int32]
    f.restype = C.c_int32
    assert f(mm._ctx, value) == 0, name


def sm_count():
    from mesh_navigation_b200 import _lib
    if _lib.LIB_PATH.endswith("libmeshnav_emu.so"):
        return int(os.environ["MNB_EMU_SMS"])
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fuzz(name):
    return np.load(os.path.join(os.path.dirname(__file__), "golden", f"fuzz_{name}.npz"))


class Plan:
    """One mesh with its costs, a CVP goal (+ robot face) and a Dijkstra seed (+ robot vertex); oracle results and the GPU's
    default-configuration results are computed once and cached."""

    def __init__(self, api, om, pos, faces, vc, w, inv, sf, sp, rf, cl):
        self.api, self.om = api, om
        self.pos, self.faces, self.vc, self.w, self.inv = pos, faces, vc, w, inv
        self.sf, self.sp, self.rf, self.cl = sf, sp, rf, cl
        self.sv = int(faces[sf][0])
        self.rv = int(faces[rf][0]) if rf >= 0 else int(faces[centre_seed(pos, faces, (0.7, 0.6))[1]][0])
        fin = w[(w > 0) & np.isfinite(w)].astype(np.float64)
        self.hop = float(np.float32(1.35) * np.float32(fin.sum() / fin.size))      # 1.35 x mean finite edge weight, as mnb_set_costs
        self._cache = {}

    def band(self, name):
        """band_delta of a named band width; None keeps the width derived from the edge weights"""
        if name == "half_hop":
            return 0.5 * self.hop              # no sweeps are derived below 2.8 hops
        if name == "odd":
            return 3.2 * self.hop              # derives 3 sweeps
        if name == "wide":
            d = self.ref("dijkstra", False)["dist"]
            return 2.0 * float(d[np.isfinite(d)].max()) + 1.0
        return None

    def ref(self, kind, robot):
        key = ("ref", kind, robot)
        if key not in self._cache:
            inv = self.inv
            if kind == "cvp":
                self._cache[key] = self.om.cvp(self.w, self.vc, self.sf, self.sp, self.rf if robot else -1, invalid=inv, cost_limit=self.cl)
            else:
                self._cache[key] = self.om.dijkstra(self.w, self.vc, self.sv, self.rv if robot else -1, invalid=inv, cost_limit=self.cl)
        return self._cache[key]

    def default(self, kind, robot):
        key = ("gpu", kind, robot)
        if key not in self._cache:
            self._cache[key] = self.run(kind, robot)
        return self._cache[key]

    def run(self, kind, robot, band="default", cluster=0, threads=0, sweeps=None):
        api = self.api
        mm = api.MeshMap(self.pos, self.faces)
        try:
            mm.setCosts(self.vc, self.w, self.inv)
            delta = self.band(band)
            if delta is not None or cluster or threads:
                mm.set_tuning(delta or 0.0, cluster, threads)
            if sweeps is not None:
                _debug(mm, "mnb_debug_set_sweeps", sweeps)
            if kind == "cvp":
                return api.CVPMeshPlanner(mm, cost_limit=self.cl).waveFrontPropagation(self.sf, self.sp, self.rf if robot else -1)
            return api.DijkstraMeshPlanner(mm, cost_limit=self.cl).dijkstra(self.sv, self.rv if robot else -1)
        finally:
            mm.close()


def _make_plan(api, om_mod, name):
    if name in FUZZ:
        d = _fuzz(name)
        pos, faces = d["pos"], d["faces"]
        inv = d["inv"] if d["inv"].size else None
        return Plan(api, om_mod.OracleMesh(pos, faces), pos, faces, d["vc"], d["w"], inv, int(d["sf"]), d["sp"], int(d["rf"]), float(d["cl"]))
    if name == "noncausal_terrain":
        # the cost-weighted terrain of test_gpu_parity.py::test_cvp_cost_weighted_non_causal with edge cost factor 2, at 160 x 160
        # so that the one-CTA kernels cross it at half a hop of band in seconds on the interpreter as well
        pos, faces = mesh_case(160, True)
        om = om_mod.OracleMesh(pos, faces)
        rng = np.random.default_rng(5)
        vc = np.where(rng.random(om.V) < 0.04, 1.2, rng.random(om.V) * 0.7).astype(np.float32)
        v, f, sp = centre_seed(pos, faces, (0.3, 0.35))
        vc[faces[f]] = 0.1
        w = om.edge_weights(vc, om.edge_distances(), 2.0)
        return Plan(api, om, pos, faces, vc, w, None, f, sp, -1, 1.0)
    if name == "delaunay_hub":
        # irregular mesh with a degree-24 hub (ELL overflow and the rescanning replay); the goal is a face of the hub
        pos, faces = delaunay_mesh(3000)
        om = om_mod.OracleMesh(pos, faces)
        vc = (np.random.default_rng(9).random(om.V) * 0.6).astype(np.float32)
        w = om.edge_weights(vc, om.edge_distances(), 1.0)
        f = face_of_vertex(faces, om.V - 1)
        return Plan(api, om, pos, faces, vc, w, None, f, pos[faces[f]].mean(0).astype(np.float32), -1, 1.0)
    raise KeyError(name)


@pytest.fixture(scope="module")
def plans(api, oracle_mod):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _make_plan(api, oracle_mod, name)
        return cache[name]
    return get


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def check_cvp(got, ref, base, what):
    assert got["outcome"] == ref["outcome"], what
    nd = int((_bits(got["dist"]) != _bits(ref["dist"])).sum())
    assert nd == 0, f"{what}: {nd} potentials differ from the oracle"
    assert (got["pred"] == ref["pred"]).all(), f"{what}: predecessors differ from the oracle"
    assert (got["cutting_face"] == ref["cutting_face"]).all(), f"{what}: cutting faces differ from the oracle"
    gd, rd = got["direction"], ref["direction"]
    assert (np.isnan(gd) == np.isnan(rd)).all(), what
    ok = ~np.isnan(rd)
    assert np.abs(gd[ok] - rd[ok]).max(initial=0.0) <= 1e-5, f"{what}: directions differ from the oracle"
    for k in ("dist", "pred", "direction", "cutting_face"):
        assert (_bits(got[k]) == _bits(base[k])).all(), f"{what}: {k} differs from the default configuration's"
    assert got["outcome"] == base["outcome"], what


def check_dijkstra(got, ref, base, what):
    assert got["outcome"] == ref["outcome"] == base["outcome"], what
    nd = int((_bits(got["dist"]) != _bits(ref["dist"])).sum())
    assert nd == 0, f"{what}: {nd} distances differ from the oracle"
    assert (got["pred"] == ref["pred"]).all(), f"{what}: predecessors differ from the oracle"
    assert (_bits(got["dist"]) == _bits(base["dist"])).all() and (got["pred"] == base["pred"]).all(), \
        f"{what}: differs from the default configuration's"


# ---- 1. CVP on the whole grid (k_cvp_grid): block size x in-round sweeps x band width ----------------------------------
@pytest.mark.parametrize("threads", THREADS)
@pytest.mark.parametrize("name", PLANS)
def test_cvp_grid_threads_sweeps_bands(plans, name, threads):
    """every threads x sweeps pair on every plan; all four bands for each pair on FULL, a rotating band elsewhere"""
    p = plans(name)
    ref, base = p.ref("cvp", True), p.default("cvp", True)
    for i, sweeps in enumerate(CVP_SWEEPS):
        bands = BANDS if name == FULL else (BANDS[(i + THREADS.index(threads)) % len(BANDS)],)
        for band in bands:
            got = p.run("cvp", True, band=band, cluster=-1, threads=threads, sweeps=sweeps)
            check_cvp(got, ref, base, (name, "grid", threads, sweeps, band))


# ---- 2. CVP on one cluster (k_cvp<CS>, MNB_CVP_THREADS per CTA) ----------------------------------------------------------
@pytest.mark.parametrize("cluster", CLUSTERS)
@pytest.mark.parametrize("name", PLANS)
def test_cvp_cluster_kernels_bands(plans, name, cluster):
    p = plans(name)
    ref, base = p.ref("cvp", True), p.default("cvp", True)
    for band in BANDS:
        got = p.run("cvp", True, band=band, cluster=cluster)
        check_cvp(got, ref, base, (name, cluster, band))


# ---- 3. Dijkstra: k_dijkstra_grid (sweeps x bands) and k_dijkstra<CS> (cluster size x block size) ------------------------
@pytest.mark.parametrize("robot", [False, True])
@pytest.mark.parametrize("name", PLANS)
def test_dijkstra_grid_sweeps_bands(plans, name, robot):
    p = plans(name)
    ref, base = p.ref("dijkstra", robot), p.default("dijkstra", robot)
    for sweeps in DIJKSTRA_SWEEPS:
        for band in BANDS:
            got = p.run("dijkstra", robot, band=band, cluster=-1, sweeps=sweeps)
            check_dijkstra(got, ref, base, (name, robot, sweeps, band))


@pytest.mark.parametrize("robot", [False, True])
@pytest.mark.parametrize("name", PLANS)
def test_dijkstra_cluster_kernels_threads(plans, name, robot):
    p = plans(name)
    ref, base = p.ref("dijkstra", robot), p.default("dijkstra", robot)
    for i, cluster in enumerate(CLUSTERS):
        for j, threads in enumerate(THREADS):
            band = BANDS[(i + j) % len(BANDS)]
            got = p.run("dijkstra", robot, band=band, cluster=cluster, threads=threads)
            check_dijkstra(got, ref, base, (name, robot, cluster, threads, band))


# ---- 4. inflation wave (k_inflate): block size x clean-candidate skip ---------------------------------------------------
def _inflation_input(name):
    if name == "delaunay_hub_disc":
        # a lethal patch just outside the hub's ring: the hub's label takes all 24 of its faces into account
        pos, faces = delaunay_mesh(3000, seed=11)
        c = pos[pos.shape[0] - 1, :2] + 0.42 * np.array([np.cos(0.3), np.sin(0.3)])
        le = np.where(np.linalg.norm(pos[:, :2] - c, axis=1) < 0.17)[0].astype(np.uint32)
        return pos, faces, le, 1.2, None
    d = _fuzz(name)
    inv = d["inv"] if "inv" in d.files and d["inv"].size else None
    return d["pos"], d["faces"], d["le"], float(d["rad"]), inv


@pytest.mark.parametrize("name", ["inflation_backstep", "inflation_never_fixed", "delaunay_hub_disc"])
def test_inflation_threads_and_skip(api, oracle_mod, name):
    pos, faces, le, rad, inv = _inflation_input(name)
    om = oracle_mod.OracleMesh(pos, faces)
    ref = om.inflation(om.edge_distances(), le, invalid=inv, inflation_radius=rad, with_vectors=True)
    assert np.abs(ref["vectors"]).sum() > 0

    def run(threads, skip):
        mm = api.MeshMap(pos, faces)
        try:
            if threads:
                mm.set_tuning(0.0, 0, threads)
            if skip is not None:
                _debug(mm, "mnb_debug_set_infl_skip", skip)
            il = api.InflationLayer(mm, inflation_radius=rad)
            got = il.waveCostInflation(le, inv)
            got["vectors"] = il.vectorMap()
            return got
        finally:
            mm.close()

    base = run(0, None)
    for threads in THREADS:
        for skip in (0, 1):
            got = run(threads, skip)
            what = (name, threads, skip)
            assert (_bits(got["dist"]) == _bits(ref["dist"])).all(), f"{what}: distances differ from the oracle"
            assert (np.isnan(got["cost"]) == np.isnan(ref["cost"])).all(), what
            ok = ~np.isnan(ref["cost"])
            assert (_bits(got["cost"][ok]) == _bits(ref["cost"][ok])).all(), f"{what}: costs differ from the oracle"
            assert (_bits(got["vectors"]) == _bits(ref["vectors"])).all(), f"{what}: vectors differ from the oracle"
            for k in ("dist", "cost", "vectors"):
                assert (_bits(got[k]) == _bits(base[k])).all(), f"{what}: {k} differs from the default configuration's"


# ---- 5. capacity edges of the round engine ---------------------------------------------------------------------------
# With no in-round sweeps every evaluation is one main-pass evaluation of a list entry, so recomputes / rounds is a lower
# bound on the mean candidate-list length; a mean above a threshold proves that at least one round's list exceeded it.
# A band wider than the mesh keeps about 0.09-0.13 V (CVP) / 0.06 V (Dijkstra) vertices in flight per round on a terrain with a
# central goal, the lower figures on multi-million-vertex terrains; the size search starts from such an estimate and grows the
# terrain by 15 % until the bound is met.

def _terrain_plan(api, oracle_mod, n):
    pos, faces = mesh_case(n, True)
    om = oracle_mod.OracleMesh(pos, faces)
    ed = om.edge_distances()
    v, f, sp = centre_seed(pos, faces)
    return Plan(api, om, pos, faces, np.zeros(om.V, np.float32), ed, None, f, sp, -1, 1.0)


def _mean_list(p, kind, cluster):
    got = p.run(kind, False, band="wide", cluster=cluster, sweeps=0)
    return got, got["recomputes"] / max(got["rounds"], 1)


def _sized_plan(api, oracle_mod, kind, cluster, threshold, per_vertex):
    n = int(math.ceil(1.02 * math.sqrt(threshold / per_vertex)))
    for _ in range(6):
        p = _terrain_plan(api, oracle_mod, n)
        first, mean = _mean_list(p, kind, cluster)
        print(f"\n{kind} cluster {cluster}: terrain {n} x {n} ({p.om.V} vertices), mean list per round >= {mean:.0f} "
              f"vs threshold {threshold}")
        if mean > threshold:
            return p, first, mean
        n = int(math.ceil(n * 1.15))
    pytest.fail(f"no terrain up to {n} x {n} gives a {kind} list above {threshold} per round")


def _capacity_case(api, oracle_mod, kind, cluster, threshold, per_vertex):
    p, first, mean = _sized_plan(api, oracle_mod, kind, cluster, threshold, per_vertex)
    assert mean > threshold
    ref = p.ref(kind, False)
    check = check_cvp if kind == "cvp" else check_dijkstra
    check(first, ref, first, (kind, cluster, "sweeps 0"))
    base = p.default(kind, False)
    check(first, ref, base, (kind, cluster, "sweeps 0 vs default"))
    if cluster == -1:
        for sweeps in (-1, 12):
            got = p.run(kind, False, band="wide", cluster=-1, sweeps=sweeps)
            check(got, ref, first, (kind, "wide band", sweeps))


def test_capacity_grid_cvp_sweep_slots(api, oracle_mod):
    """k_cvp_grid with more than 2 x SM x SW_CAP candidates per round: the one-thread main pass walks a CTA's share in SW_CAP
    chunks, stage slots past SW_CAP are not swept, and delta_r is narrowed for the long front"""
    _capacity_case(api, oracle_mod, "cvp", -1, 2 * sm_count() * SW_CAP, 0.12)


def test_capacity_grid_dijkstra_sweep_slots(api, oracle_mod):
    _capacity_case(api, oracle_mod, "dijkstra", -1, 2 * sm_count() * SW_CAP, 0.06)


def test_capacity_one_cta_stage_overflow(api, oracle_mod):
    """k_cvp<1> and k_dijkstra<1>: one CTA stages a whole round's list, more than 2 x Stage::CAP entries, so stage_put
    sends the overflow straight to the global list"""
    _capacity_case(api, oracle_mod, "cvp", 1, 2 * STAGE_CAP, 0.115)
    _capacity_case(api, oracle_mod, "dijkstra", 1, 2 * STAGE_CAP, 0.06)


def test_capacity_grid_stage_overflow_large_mesh(api, oracle_mod):
    """k_cvp_grid with more than SM x Stage::CAP evaluations per round: some CTA stages past Stage::CAP in some round
    (a multi-million-vertex terrain on an H100; not run on the interpreter)"""
    _capacity_case(api, oracle_mod, "cvp", -1, sm_count() * STAGE_CAP, 0.12)
