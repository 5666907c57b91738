"""Drives every kernel outside the timed solve step once at benchmark scale, so that one ncu metric pass gives their
duration and DRAM traffic:

    ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none \
        -k regex:'preintegrate|marg|outlier|triangulate|shift_depth|projection_eval|imu_leg_eval|prior_eval' --csv \
        python tools/aux_kernels.py [NW] [F]

preintegrate_kernel: NW * 10 intervals x 33 samples (the set-up of one batch of windows); outlier / triangulate /
shift_depth: the resident NW x F batch after a solve; marg kernels: NW windows at m = 19 + F, n = 86.
"""
import os
import sys
import time
import ctypes as C
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cerberus_b200 import abi, lib, synth      # noqa: E402

NW = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
F = int(sys.argv[2]) if len(sys.argv) > 2 else 150


def wall(fn, reps=3):
    best = 1e9
    for _ in range(reps):
        t = time.perf_counter(); fn(); best = min(best, time.perf_counter() - t)
    return best


def main():
    cfg = abi.default_config(); cfg.max_batch = NW; cfg.max_features = 160; cfg.max_obs = 160 * 11
    be = lib.Backend(cfg)
    small, truth = synth.generate_batch(8, F, be, prior_features=24, return_truth=True)
    big = synth.tile_batch(small, NW)
    # preintegration at scale: the 8 x 11 raw jobs repeated to NW * 10 intervals
    pcfg = abi.default_preint_config()
    nj = NW * 10
    jobs = (abi.PreintJob * nj)()
    src = truth.raw_jobs
    for k in range(nj):
        C.memmove(C.byref(jobs[k]), C.byref(src[k % len(src)]), C.sizeof(abi.PreintJob))
    t = wall(lambda: be.preintegrate(pcfg, jobs, nj))
    print(f"preintegrate_batch (host buffers in/out): {nj} intervals x 33 samples: {t * 1e3:.2f} ms wall = {nj / t:.0f} intervals/s")
    be.upload(big); be.solve_resident(); be.sync()
    t = wall(lambda: be.outlier_errors(NW)); print(f"outlier_errors ({NW} x {F}): {t * 1e3:.2f} ms wall")
    t = wall(lambda: be.triangulate(NW)); print(f"triangulate    ({NW} x {F}): {t * 1e3:.2f} ms wall")
    t = wall(lambda: be.shift_depth(NW)); print(f"shift_depth    ({NW} x {F}): {t * 1e3:.2f} ms wall")
    # per-frame use (BASELINE.json configs[2]: one window per camera frame): latency of the drop-in call for ONE window, host buffers in / out
    one = synth.tile_batch(small, 1)
    saved1 = one.copy_states()
    def solve_one():
        one.restore_states(saved1); be.solve_batch(one)
    t = wall(solve_one, reps=5); ms, _ = be.last_solve_stats()
    print(f"cerb_solve_window (1 window x {F} features, 12 iterations, host buffers in / out): {t * 1e3:.2f} ms wall, {ms:.2f} ms on the device")
    be.upload(big); be.solve_resident(); be.sync()
    rng = np.random.default_rng(0)
    m, n = 19 + F, 86
    pos = m + n
    nwm = min(NW, 296)
    J = rng.standard_normal((nwm, 3 * pos, pos)); J[:, :, :m] *= np.exp(rng.uniform(-2, 2, (nwm, 1, m)))
    A = np.swapaxes(J, 1, 2) @ J; b = (np.swapaxes(J, 1, 2) @ rng.standard_normal((nwm, 3 * pos, 1)))[..., 0]
    t = wall(lambda: be.marginalize_schur(A, b, m), reps=2)
    print(f"marginalize_schur ({nwm} windows, m={m}, n={n}): {t * 1e3:.2f} ms wall = {t / nwm * 1e6:.1f} us / window")
    # the whole marginalization step on the resident batch (assembly by the solver's linearisation passes + eigen Schur complement), host buffers out
    flags = np.zeros(NW, dtype=np.int32)
    J = np.zeros((NW, abi.MAX_PRIOR_DIM * abi.MAX_PRIOR_DIM)); r = np.zeros((NW, abi.MAX_PRIOR_DIM))
    priors = (abi.Prior * NW)()
    for w in range(NW):
        priors[w].linearized_jacobians = J[w].ctypes.data_as(abi.c_dp); priors[w].linearized_residuals = r[w].ctypes.data_as(abi.c_dp)
    sw = be.batch_marginalize(flags, None, priors)
    t = wall(lambda: be.batch_marginalize(flags, None, priors), reps=2)
    print(f"batch_marginalize ({NW} windows x {F} features anchored at frame 0: m = {19 + F}, n = {priors[0].n}; MARGIN_OLD at the solved states): {t * 1e3:.2f} ms wall = {t / NW * 1e6:.1f} us / window, "
          f"Jacobi sweeps {sw[:, 0].mean():.1f} / {sw[:, 1].mean():.1f}")


if __name__ == "__main__":
    main()
