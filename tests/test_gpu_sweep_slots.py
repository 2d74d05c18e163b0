"""The whole-grid single-plan kernels (k_cvp_grid, k_dijkstra_grid) at GridStage capacities from one slot per CTA to past the
default, set through mnb_debug_set_sweep_slots.

The capacity decides how many staged candidates a CTA keeps in shared memory (the rest go straight to the global list), how
many take part in the in-round sweeps, the chunks of the one-thread main pass and the band narrowing of long fronts; it is
set before the weights are installed, so the single-plan band widths derived from it change with it as well.  None of that
may change a result: every run is compared with the oracle (potentials and distances bit for bit, predecessors and cutting
faces exactly, CVP directions within 1e-5) and with the default capacity's run of the same plan, all outputs bit for bit.
A resumed mnb_cvp_replan is compared with a fresh plan at each capacity.  The GPU tests run with -m gpu on an H100; the last
test replays them on the CPU interpreter of the kernels (tests/emu)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gpu_launch_configs import _terrain_plan, check_cvp, check_dijkstra, plans, sm_count  # noqa: F401  (plans: fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANS = ("deep_cascade_planar", "deep_cascade_delaunay", "cutoff_cascade", "seed_after_neighbour", "noncausal_terrain",
         "delaunay_hub")
SLOTS = (1, 7, 64, 1000, 4096, 7000)         # 7000 x GRID_SLOT_BYTES: most of an H100's 227 KB of shared memory per block
SWEEPS = (-1, 0, 1, 5, 24, 64)               # -1: derived from the band width


@pytest.fixture(scope="module")
def api():
    from mesh_navigation_b200 import api as A
    return A


def _hook(mm, name, value):
    f = getattr(mm.L, name)
    f.argtypes = [C.c_void_p, C.c_int32]
    f.restype = C.c_int32
    return f(mm._ctx, value)


def _map(api, p, slots, sweeps, band=None):
    """a map of plan p with `slots` GridStage slots (0: the default), set before the weights so that the derived bands
    follow them, unless `band` (a name of Plan.band) fixes the band"""
    mm = api.MeshMap(p.pos, p.faces)
    assert _hook(mm, "mnb_debug_set_sweep_slots", slots) == 0, slots
    mm.setCosts(p.vc, p.w, p.inv)
    if band is not None:
        mm.set_tuning(p.band(band), 0, 0)
    if sweeps is not None:
        assert _hook(mm, "mnb_debug_set_sweeps", sweeps) == 0
    return mm


def _run(api, p, kind, robot, slots, sweeps=None, band=None):
    mm = _map(api, p, slots, sweeps, band)
    try:
        if kind == "cvp":
            return api.CVPMeshPlanner(mm, cost_limit=p.cl).waveFrontPropagation(p.sf, p.sp, p.rf if robot else -1)
        return api.DijkstraMeshPlanner(mm, cost_limit=p.cl).dijkstra(p.sv, p.rv if robot else -1)
    finally:
        mm.close()


@pytest.mark.gpu
def test_sweep_slots_hook_arguments(api, plans):
    p = plans("cutoff_cascade")
    mm = api.MeshMap(p.pos, p.faces)
    try:
        for bad in (-1, 65536, 1 << 30):                  # (65535 slots, the most a uint16_t dirty list indexes, exceed 227 KB)
            assert _hook(mm, "mnb_debug_set_sweep_slots", bad) != 0, bad
        for ok in (0, 1, 7000):
            assert _hook(mm, "mnb_debug_set_sweep_slots", ok) == 0, ok
    finally:
        mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("slots", SLOTS)
@pytest.mark.parametrize("name", PLANS)
def test_cvp_grid_sweep_slots(api, plans, name, slots):
    """k_cvp_grid with the goal cutoff armed and without, at two sweep counts per capacity (rotating over SWEEPS)"""
    p = plans(name)
    k = SLOTS.index(slots)
    for robot in (True, False):
        ref, base = p.ref("cvp", robot), p.default("cvp", robot)
        for sweeps in (SWEEPS[k % len(SWEEPS)], SWEEPS[(k + 3 + robot) % len(SWEEPS)]):
            got = _run(api, p, "cvp", robot, slots, sweeps)
            check_cvp(got, ref, base, (name, "slots", slots, "sweeps", sweeps, "robot", robot))


@pytest.mark.gpu
@pytest.mark.parametrize("slots", SLOTS)
@pytest.mark.parametrize("name", PLANS)
def test_dijkstra_grid_sweep_slots(api, plans, name, slots):
    p = plans(name)
    k = SLOTS.index(slots)
    for robot in (False, True):
        ref, base = p.ref("dijkstra", robot), p.default("dijkstra", robot)
        sweeps = SWEEPS[(k + robot) % len(SWEEPS)]
        got = _run(api, p, "dijkstra", robot, slots, sweeps)
        check_dijkstra(got, ref, base, (name, "slots", slots, "sweeps", sweeps, "robot", robot))


@pytest.mark.gpu
def test_sweep_slots_overflow_to_global(api, plans, oracle_mod):
    """one slot per CTA and a band wider than the mesh: with no sweeps every evaluation is a main-pass evaluation of a list
    entry, so recomputes / rounds bounds the mean list from below; a mean above one entry per CTA proves that CTAs staged
    past their slot, and the stage overflowed into the global list"""
    p = plans("seed_after_neighbour")
    got = _run(api, p, "cvp", False, 1, 0, "wide")
    assert got["recomputes"] / max(got["rounds"], 1) > sm_count(), (got["recomputes"], got["rounds"])
    check_cvp(got, p.ref("cvp", False), p.default("cvp", False), ("overflow", 1))
    p = _terrain_plan(api, oracle_mod, 100)        # (the fixture's cost limit stops its Dijkstra wave after a few vertices)
    got = _run(api, p, "dijkstra", False, 1, 0, "wide")
    assert got["recomputes"] / max(got["rounds"], 1) > sm_count(), (got["recomputes"], got["rounds"])
    check_dijkstra(got, p.ref("dijkstra", False), p.default("dijkstra", False), ("overflow", 1))


def _replan_chain(api, p, slots):
    """a plan, then three rounds of cost changes at several depths of its pop order, each followed by a resumed
    mnb_cvp_replan (k_cvp_grid<true>) and a fresh plan on the same costs; returns the (replan, fresh plan) pairs"""
    mm = _map(api, p, slots, None)
    try:
        pl = api.CVPMeshPlanner(mm, cost_limit=p.cl)
        vc = p.vc.copy()
        out = [(pl.waveFrontReplan(p.sf, p.sp, p.rf, np.empty(0, np.uint32)), None)]
        d = out[0][0]["dist"]
        fin = np.where(np.isfinite(d))[0]
        order = fin[np.argsort(d[fin], kind="stable")]
        for k, q in enumerate((0.2, 0.5, 0.8)):
            ch = order[int(q * (order.size - 1)):][:4].astype(np.uint32)
            vals = ((vc[ch] + 0.05 * (k + 1)) % p.cl).astype(np.float32)
            mm.layerChanged(ch, vals, 1.0)
            vc[ch] = vals
            got = pl.waveFrontReplan(p.sf, p.sp, p.rf, ch)
            out.append((got, pl.waveFrontPropagation(p.sf, p.sp, p.rf)))
        return out
    finally:
        mm.close()


@pytest.mark.gpu
@pytest.mark.parametrize("slots", (1, 64, 4096))
def test_cvp_replan_sweep_slots(api, plans, slots):
    """each resumed replan equals the fresh plan on the same costs, and both equal the default capacity's, bit for bit"""
    p = plans("deep_cascade_delaunay")
    base, got = _replan_chain(api, p, 0), _replan_chain(api, p, slots)
    check_cvp(got[0][0], p.ref("cvp", True), base[0][0], ("first plan", slots))
    resumed = 0
    for i in range(1, len(got)):
        check_cvp(got[i][0], got[i][1], base[i][0], ("replan", slots, i))
        check_cvp(got[i][1], got[i][1], base[i][1], ("fresh plan", slots, i))
        resumed += got[i][0]["settled"] < got[i][1]["settled"]
    assert resumed >= 1, resumed


@pytest.mark.parametrize("shuffle", [None, "4"])
def test_sweep_slots_on_the_cpu_interpreter(shuffle):
    """the GPU tests above with the kernels compiled by g++ against tests/emu, on 4 emulated SMs; once in the default warp
    order, once in a randomised one"""
    runner = os.path.join(ROOT, "tests", "emu", "run_suite.py")
    me = os.path.abspath(__file__)
    env = dict(os.environ, MNB_EMU_SMS="4", **({"MNB_EMU_SHUFFLE": shuffle} if shuffle else {}))
    r = subprocess.run([sys.executable, runner, me, "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, f"shuffle {shuffle}:\n{tail}"
