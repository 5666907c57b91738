"""Per-phase cycle breakdown of vilo_solve_kernel (profiling build: `make prof`, -DCERB_PHASE_TIMING).
Usage: python tools/phase_profile.py [NW] [F] [REP] -> prints cycles per window per phase and shares."""
import sys, os, ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from cerberus_b200 import abi, synth, lib
NW = int(sys.argv[1]) if len(sys.argv) > 1 else 132
F = int(sys.argv[2]) if len(sys.argv) > 2 else 150
REP = int(sys.argv[3]) if len(sys.argv) > 3 else 2
NAMES = {0: "zero+geometry", 1: "vision_linearize (total)", 2: "inertial_linearize (total)", 3: "post-linearize (sums, symmetrise, scaling)",
         4: "dogleg diag + Cauchy", 5: "Schur/Hyy join wait (warp0 after 6)", 6: "Hyy chain Cholesky (warp 0)", 7: "lambda Schur DMMA (warp 1)",
         8: "T = L^-1 Hyx", 9: "S - T T^T DMMA", 10: "dense Cholesky 79 (rest; panels in 44-47)", 11: "back-substitution x", 12: "y part (warp 0)", 13: "inverse depths (warp 0 waits)",
         14: "gn norms + dogleg scalars + step", 15: "apply_plus + geometry", 16: "vision_cost", 17: "inertial_cost + prior", 18: "accept / copy",
         20: "  vis: chunk setup", 21: "  vis: eval + tile write", 22: "  vis: DMMA Gram + partial store", 23: "  vis: reduce + scatter", 24: "  vis: per-feature tail",
         28: "    dmma loop (warp 0 view)", 29: "    partial stores + W (warp 0)", 30: "  imu: warps 0-2 (factor rounds, tail)", 32: "    imu warp 0: zero + expand Ju", 33: "    imu warp 0: whiten", 34: "    imu warp 0: S prefetch + Gram", 35: "    imu warp 0: scatter", 36: "    imu warp 0: round barrier", 31: "  imu: warps 3-7 (prior)",
         19: "  schur (warp 1): rhs + Cauchy v^T H v", 37: "  schur (warp 1): sinv + block table + first fetch", 38: "  schur (warp 1): tile scale/store + barrier (all tiles)", 39: "  schur (warp 1): DMMA loop + barrier (all tiles)",
         25: "  imu: linearize (10 threads)", 26: "  imu: whiten + Gram x10", 27: "  imu: prior",
         47: "  chol: first diag block + panel solve + barrier", 44: "  chol: warp 0 next diag block (update + factor)", 45: "  chol: trailing update (warp 1)",
         46: "  chol: warp 0 wait at the panel barrier",
         43: "  bsub: inverse depths (warp 1)"}
cfg = abi.default_config(); cfg.max_batch = NW; cfg.max_features = 160; cfg.max_obs = 160 * 11
gb = lib.Backend(cfg, lib_path=os.path.join(ROOT, "tools", "libcerberus_b200_prof.so"))
batch = synth.generate_batch(min(NW, 8), F, gb, prior_features=24)
big = synth.tile_batch(batch, NW)
gb.upload(big)
buf = (C.c_ulonglong * 48)()
gb.lib.cerb_prof_phase_cycles.argtypes = [C.POINTER(C.c_ulonglong)]
for rep in range(REP):
    gb.lib.cerb_prof_phase_cycles(buf)
    gb.solve_resident(); gb.sync()
    ms, _ = gb.last_solve_stats()
    gb.lib.cerb_prof_phase_cycles(buf)
    v = np.array(list(buf), dtype=np.float64) / NW
    top = sum(v[k] for k in range(0, 19))
    print(f"rep {rep}: {ms:.3f} ms for {NW} windows; {top:.0f} cycles per window in top-level phases")
    for k in sorted(NAMES):
        if v[k] > 0: print(f"  [{k:2d}] {NAMES[k]:48s} {v[k]:12.0f} cyc  {100 * v[k] / top:5.1f} %")
