"""Dev script (GPU box): A/B of batch-kernel builds / cluster sizes / band widths on the config-4 mesh.
  python tools/gpu_batch2.py <grid side> <spec> [<spec> ...]      spec = lib:cluster:goals:delta
lib = path of a libmeshnav_b200.so build ('-' = the in-tree one); one subprocess per spec (a process loads one build).
Every spec prints plans/s, kernel ms, rounds and recomputes per plan, and a checksum of the potentials (all builds must agree)."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

def worker(n, lib, cs, ng, delta):
    sys.path.insert(0, ROOT)
    from mesh_navigation_b200 import _lib
    if lib != "-": _lib.LIB_PATH = os.path.join(ROOT, lib)
    import time, zlib, numpy as np, torch
    from mesh_navigation_b200 import synth
    from mesh_navigation_b200.api import MeshMap
    pos, faces = synth.grid_mesh(n, n, terrain=True, seed=42)
    mm = MeshMap(pos, faces); mm.setCosts(np.zeros(mm.V, np.float32), mm.edgeDistances())
    goals = synth.batch_goal_vertices(mm.V, 1024, seed=1234)
    gi, gj = np.minimum(goals % n, n - 2), np.minimum(goals // n, n - 2)
    sfs = (2 * (gj * (n - 1) + gi)).astype(np.uint32); sps = pos[faces[sfs]].mean(1).astype(np.float32)
    mm.set_tuning(delta, cs, 0)
    out = torch.empty((ng, mm.V), dtype=torch.float32, device="cuda")
    mm.use_device_pointers(True)
    best = 1e9
    for rep in range(2):
        t = time.time(); mm.cvp_batch_dev(sfs[:ng], sps[:ng], 1.0, out.data_ptr()); torch.cuda.synchronize(); best = min(best, time.time() - t)
    mm.use_device_pointers(False)
    st = mm.stats()
    chk = zlib.crc32(out[: min(ng, 8)].cpu().numpy().tobytes())
    print(f"n={n} lib={lib} cluster={cs} goals={ng} delta={delta}: {best*1e3:.1f} ms -> {ng/best:.1f} plans/s, kernel {st['kernel_ms']:.1f} ms "
          f"rounds/plan {st['rounds']/ng:.0f} recomp/V {st['recomputes']/ng/mm.V:.2f} crc {chk:08x}", flush=True)

if __name__ == "__main__":
    if sys.argv[1] == "--worker":
        worker(int(sys.argv[2]), sys.argv[3], int(sys.argv[4]), int(sys.argv[5]), float(sys.argv[6]))
    else:
        n = sys.argv[1]
        for spec in sys.argv[2:]:
            f = spec.split(":")
            r = subprocess.run([sys.executable, __file__, "--worker", n, f[0], f[1], f[2], f[3]], capture_output=True, text=True, timeout=600)
            print((r.stdout.strip() or ("FAILED: " + r.stderr[-400:])), flush=True)
