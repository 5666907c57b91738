"""Per-phase cycle breakdown of the Jacobi rounds of marg_schur_kernel (profiling build: `make prof`, -DCERB_PHASE_TIMING).
Usage: python tools/marg_phase.py [windows] -> cycles per window per phase for the four sizes of tools/marg_bench.py."""
import sys, os, ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from cerberus_b200 import abi, lib
NW = int(sys.argv[1]) if len(sys.argv) > 1 else 132
NAMES = {46: "T stage loads (thread 0)", 40: "X: 2x2 blocks (thread 0)", 41: "barrier 1 (thread 0)", 42: "Y: V / T rotations (thread 0)", 43: "barrier 2 (thread 0)",
         47: "angle thread: X + barrier 1", 44: "angle thread: angles", 45: "angle thread: barrier 2"}
cfg = abi.default_config(); cfg.max_batch, cfg.max_features, cfg.max_obs = 2, 8, 88
be = lib.Backend(cfg, lib_path=os.path.join(ROOT, "tools", "libcerberus_b200_prof.so"))
be.lib.cerb_prof_phase_cycles.argtypes = [C.POINTER(C.c_ulonglong)]
buf = (C.c_ulonglong * 48)()
rng = np.random.default_rng(0)
for m, n in ((6, 80), (19 + 16, 86), (19 + 50, 86), (19 + 150, 86)):
    pos = m + n
    J = rng.standard_normal((NW, 3 * pos, pos)); J[:, :, :m] *= np.exp(rng.uniform(-2, 2, (NW, 1, m)))
    A = np.swapaxes(J, 1, 2) @ J; b = (np.swapaxes(J, 1, 2) @ rng.standard_normal((NW, 3 * pos, 1)))[..., 0]
    be.marginalize_schur(A[:2], b[:2], m)
    be.lib.cerb_prof_phase_cycles(buf)
    _, _, sw = be.marginalize_schur(A, b, m, return_sweeps=True)
    be.lib.cerb_prof_phase_cycles(buf)
    v = np.array(list(buf), dtype=np.float64) / NW
    rounds = ((sw[:, 0] + 1) * (m + (m & 1) - 1) + (sw[:, 1] + 1) * (n + (n & 1) - 1)).mean()
    print(f"m={m} n={n}: {rounds:.0f} rounds per window; thread-0 total {sum(v[k] for k in (46, 40, 41, 42, 43)):.0f} cycles per window")
    for k in (46, 40, 41, 42, 43, 47, 44, 45):
        print(f"  [{k}] {NAMES[k]:34s} {v[k]:12.0f} cyc  {v[k] / rounds:8.0f} per round")
