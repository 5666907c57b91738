"""Generate the frozen known-answer vectors of tests/golden/*.npz with the CPU oracle.

The reference ships no golden vectors for this path.  The factor-level vectors (A1 kinematics, the three projection
factors, the IMU-leg factor incl. sqrt_info) are outputs of THE REFERENCE'S OWN SOURCES, compiled where they lie against
the header shims of oracle/shim (oracle/_ref/libcerberus_ref.so, `make -C oracle ref REF=<Cerberus checkout>/src`).
The window-level vector (a full 12-iteration solve) comes from the oracle's restatement of ceres-solver 1.14, which is
not available here.  Seeds of the inputs: the kinematics probe of src/test/ceres_test.cpp:16-18, the A1 geometry of
estimator.cpp:143-156, the perturbation of imu_leg_factor.cpp:43.  Re-run:  python tests/golden/make_golden.py
"""
import os
import sys
import ctypes as C
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from cerberus_b200 import abi, synth          # noqa: E402
from oracle_lib import OracleBackend, RefBackend           # noqa: E402
from test_oracle_jacobians import proj_inputs, imu_leg_setup   # noqa: E402


def window_arrays(batch, w=0):
    d = batch.descs[w]
    return dict(features=batch.features[w][:d.n_features].copy(), obs=batch.obs[w][:d.n_obs].copy(), preint=batch.preint[w].copy(),
                prior_J=batch.prior_J[w].copy(), prior_r=batch.prior_r[w].copy(), prior_raw=np.frombuffer(bytes(d.prior), dtype=np.uint8).copy(),
                state_raw=np.frombuffer(bytes(batch.states[w]), dtype=np.uint8).copy(), para_Feature=batch.para_Feature[w].copy())


def main():
    ob = OracleBackend()
    ref = RefBackend(live=True)         # the compiled reference sources generate the factor-level vectors
    out = {}
    # --- A1 kinematics at the probe of src/test/ceres_test.cpp:16-18, all four legs
    q = np.tile(np.array([0.1, 0.1, 0.3]), (4, 1))
    pc = abi.default_preint_config()
    fix = np.array([[pc.rho_fix[l][k] for k in range(4)] for l in range(4)])
    lc = np.full(4, 0.21)
    names = ("fk", "jac", "dfk_drho", "dJ_dq", "dJ_drho")
    for n, a in zip(names, ref.a1_kinematics(q, lc, fix)):
        out["kin_" + n] = a
    out["kin_q"], out["kin_lc"], out["kin_fix"] = q, lc, fix
    # --- projection factors
    for kind in range(3):
        args = proj_inputs(np.random.default_rng(100 + kind), 6)
        r, j = ref.eval_projection(kind, *args)
        for i, a in enumerate(args):
            out[f"proj{kind}_in{i}"] = a
        out[f"proj{kind}_res"], out[f"proj{kind}_jac"] = r, j
    # --- IMU-leg factor
    pre, params = imu_leg_setup(2)
    r, j, s = ref.eval_imu_leg(pre, params)
    out["imu_pre"], out["imu_params"], out["imu_res"], out["imu_jac"], out["imu_sqrt_info"] = pre, params, r, j, s
    # --- one small window: inputs and the solved state after 12 iterations
    batch, truth = synth.generate_batch(1, 6, ob, prior_features=4, return_truth=True, window0=424242)
    for k, v in window_arrays(batch).items():
        out["win_" + k] = v
    out["win_job0_samples"] = truth.raw_samples[0, 1].copy()          # raw IMU/leg samples of interval 0 -> 1
    out["win_job0"] = np.frombuffer(bytes(truth.raw_jobs[1]), dtype=np.uint8).copy()
    rep = ob.solve_batch(batch)
    st = batch.state_array()
    out["win_solved_pose"], out["win_solved_sb"], out["win_solved_lb"], out["win_solved_ex"] = st["para_Pose"][0].copy(), st["para_SpeedBias"][0].copy(), st["para_LegBias"][0].copy(), st["para_Ex_Pose"][0].copy()
    out["win_solved_feature"] = batch.para_Feature[0].copy()
    out["win_report"] = rep
    np.savez_compressed(os.path.join(HERE, "kat_v1.npz"), **out)
    print("wrote", os.path.join(HERE, "kat_v1.npz"), sum(v.nbytes for v in out.values()), "bytes raw")


if __name__ == "__main__":
    main()
