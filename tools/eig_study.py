"""How much does the marginalization prior -- and through it the published trajectory -- depend on the symmetric eigen-solver?
(VERDICT r1 "settle the eigen-solver question with numbers".)

The reference factors the marginalized Hessian with Eigen::SelfAdjointEigenSolver (Householder tridiagonalisation + implicit QR,
marginalization_factor.cpp:281-305) and clamps eigenvalues at eps = 1e-8.  The device kernels use Jacobi rotations.  This script
replays the same synthetic sequences (>= 20 chained frames: solve -> double2vector -> marginalize -> slide) through the CPU oracle with
   A: the oracle restatement, tridiagonal-QR eigen-solver (oracle/sym_eig_qr.h)
   B: the oracle restatement, cyclic Jacobi
   C: the reference's own MarginalizationInfo classes (oracle/_ref) on the QR solver, where oracle/_ref is present
and prints the per-frame differences of the raw solver output and of what the estimator publishes (after double2vector).

    python tools/eig_study.py [n_robots] [n_frames] [tracked]
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from cerberus_b200 import abi, synth, estimator
import oracle_lib

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4
nf = int(sys.argv[2]) if len(sys.argv) > 2 else 45
tracked = int(sys.argv[3]) if len(sys.argv) > 3 else 110
cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 256; cfg.max_obs = 256 * 11
pcfg = abi.default_preint_config()
seq = synth.generate_sequence(n, nf, tracked=tracked, max_len=16, min_len=3)
arms = {"A oracle/QR": oracle_lib.OracleOps(cfg, eig_mode=0), "B oracle/Jacobi": oracle_lib.OracleOps(cfg, eig_mode=1)}
if oracle_lib.ref_lib() is not None:
    arms["C reference classes/QR"] = oracle_lib.OracleOps(cfg, eig_mode=0, marg=oracle_lib.RefBackend(live=True))
    arms["D reference classes/Jacobi"] = oracle_lib.OracleOps(cfg, eig_mode=1, marg=oracle_lib.RefBackend(live=True))
runs = {}
for name, ops in arms.items():
    d = estimator.ReplayDriver(ops, cfg, pcfg, n, max_features=256).run(seq)
    P, R = d.poses()
    flags = None
    runs[name] = (P, R, d)
    err = np.linalg.norm(P - seq.p[:, 10:10 + P.shape[1]], axis=-1)
    print(f"{name:28s}: {P.shape[1]} frames, final position error vs truth {err[:, -1].round(3)} m, iterations of the last solve {d.reports[-1]['iterations']}")
names = list(runs)
base = names[0]
print(f"\nper-frame max |published position difference| vs '{base}' [m] (over {n} robots), and rotation difference [rad]:")
for other in names[1:]:
    dP = np.abs(runs[other][0] - runs[base][0]).max(axis=(0, 2))
    dR = np.abs(runs[other][1] - runs[base][1]).max(axis=(0, 2, 3))
    print(f"  {other}:")
    print("    pos:", " ".join(f"{v:.1e}" for v in dP))
    print("    rot:", " ".join(f"{v:.1e}" for v in dR))
    print(f"    max over the replay: {dP.max():.2e} m, {dR.max():.2e} rad")
