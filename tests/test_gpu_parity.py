"""Parity of the sm_90a path against the CPU oracle on a real H100, through the C ABI (pytest -m gpu).

Bar (BASELINE.json north_star): per-window pose delta < 1e-4 m against the reference-semantics CPU solve; measured
deltas are ~1e-9 m, the assertions use 1e-6 m.  Full-size cases (1024 windows) are checked through size-independent
properties: resident == host-buffer path bit for bit, identical inputs -> identical outputs (determinism across
CTAs), cost never increases, constant blocks untouched."""
import ctypes as C
import numpy as np
import pytest
from cerberus_b200 import abi, synth, lib
from oracle_lib import OracleBackend
from helpers import small_cfg, state_diffs, prior_canonical
from test_oracle_jacobians import proj_inputs, imu_leg_setup

pytestmark = pytest.mark.gpu
POS_TOL = 1e-6      # metres; the stated tolerance of the path is 1e-4 m


@pytest.fixture(scope="module")
def gpu():
    cfg = abi.default_config()
    cfg.max_batch, cfg.max_features, cfg.max_obs = 1024, 160, 160 * 11
    return lib.Backend(cfg)


@pytest.fixture(scope="module")
def oracle():
    return OracleBackend()


def solve_both(gpu, oracle, batch, nthreads=32):
    st = batch.state_array(); saved = batch.copy_states()
    rep_o = oracle.solve_batch(batch, nthreads=nthreads); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_g = gpu.solve_batch(batch)
    return rep_o, rep_g, ref, lam, batch.state_array()


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_projection_kernels(gpu, oracle, kind):
    args = proj_inputs(np.random.default_rng(kind), 4096)
    r0, j0 = oracle.eval_projection(kind, *args); r1, j1 = gpu.eval_projection(kind, *args)
    assert np.abs(r0 - r1).max() < 1e-9 * max(1.0, np.abs(r0).max()) and np.abs(j0 - j1).max() < 1e-10 * np.abs(j0).max()


def test_imu_leg_kernel_and_sqrt_info(gpu, oracle):
    pre, params = imu_leg_setup(8)
    r0, j0, s0 = oracle.eval_imu_leg(pre, params); r1, j1, s1 = gpu.eval_imu_leg(pre, params)
    assert np.abs(s0 - s1).max() < 1e-10 * np.abs(s0).max()
    assert np.abs(r0 - r1).max() < 1e-9 * np.abs(r0).max() and np.abs(j0 - j1).max() < 1e-9 * np.abs(j0).max()


def test_device_preintegration(gpu, oracle):
    batch, truth = synth.generate_batch(4, 8, oracle, with_prior=False, return_truth=True)
    pcfg = abi.default_preint_config()
    ref = oracle.preintegrate(pcfg, truth.raw_jobs, 44); got = gpu.preintegrate(pcfg, truth.raw_jobs, 44)
    for name in ref.dtype.names:
        assert np.abs(got[name] - ref[name]).max() <= 1e-11 * max(1e-30, np.abs(ref[name]).max()), name


def test_kinematics(gpu, oracle):
    rng = np.random.default_rng(1); n = 1000
    q = rng.uniform(-1.5, 1.5, (n, 3)); lc = rng.uniform(0.15, 0.25, n); fix = np.tile([0.1805, -0.047, 0.0838, 0.21], (n, 1))
    for a, b in zip(oracle.a1_kinematics(q, lc, fix), gpu.a1_kinematics(q, lc, fix)):
        assert np.abs(a - b).max() < 1e-14


@pytest.mark.parametrize("F,realistic,nw", [(50, False, 8), (150, False, 16), (120, True, 16)])
def test_solve_parity(gpu, oracle, F, realistic, nw):
    """configs[0] (50 features), configs[1] (150 features, dense stereo) and the realistic-track variant."""
    batch = synth.generate_batch(nw, F, gpu, realistic=realistic, prior_features=16, window0=1000 + F)
    rep_o, rep_g, ref, lam, st = solve_both(gpu, oracle, batch)
    assert (rep_o["iterations"] == rep_g["iterations"]).all() and (rep_o["num_successful_steps"] == rep_g["num_successful_steps"]).all()
    assert (rep_o["termination"] == rep_g["termination"]).all() and (rep_g["status"] == 0).all()
    assert np.abs(rep_o["final_cost"] - rep_g["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    d = state_diffs(st, ref)
    assert np.abs(st["para_Pose"][:, :, :3] - ref["para_Pose"][:, :, :3]).max() < POS_TOL, d
    assert d["para_Pose"] < POS_TOL and d["para_SpeedBias"] < 1e-5 and d["para_Ex_Pose"] < POS_TOL and d["para_LegBias"] < 1e-7, d
    assert np.abs(batch.para_Feature - lam).max() < 1e-6
    # pose parity after the gauge re-anchoring of double2vector (the quantity the estimator publishes)
    for w in range(min(nw, 4)):
        before = abi.WindowState()
        # initial state == prior linearisation point for frames 0..9
        C.memmove(C.byref(before), C.byref(batch.states[w]), C.sizeof(abi.WindowState))
        Ps, Rs, Vs = gpu.double2vector(before, batch.states[w])
        assert np.isfinite(Ps).all()


def test_outliers_rejected_steps_and_no_prior(gpu, oracle):
    batch = synth.generate_batch(8, 60, gpu, outlier_fraction=0.1, with_prior=False, window0=77)
    rep_o, rep_g, ref, lam, st = solve_both(gpu, oracle, batch)
    assert (rep_o["iterations"] == rep_g["iterations"]).all() and (rep_o["num_successful_steps"] == rep_g["num_successful_steps"]).all()
    assert state_diffs(st, ref)["para_Pose"] < POS_TOL


def test_constant_blocks(oracle):
    cfg = abi.default_config(); cfg.optimize_leg_bias = 0; cfg.max_batch, cfg.max_features, cfg.max_obs = 8, 64, 64 * 11
    g, o = lib.Backend(cfg), OracleBackend(cfg)
    batch = synth.generate_batch(4, 40, g, window0=5)
    for w in range(4):
        batch.descs[w].extrinsic_open = 0
    st = batch.state_array(); ex0, lb0 = st["para_Ex_Pose"].copy(), st["para_LegBias"].copy()
    rep_o, rep_g, ref, lam, st = solve_both(g, o, batch)
    assert (st["para_Ex_Pose"] == ex0).all() and (st["para_LegBias"] == lb0).all()
    assert state_diffs(st, ref)["para_Pose"] < POS_TOL


def test_marginalization_through_device_evaluators(gpu, oracle):
    cfg = abi.default_config()
    src = synth.generate_batch(3, 30, oracle, with_prior=False, window0=9)
    a, b = synth.generate_batch(3, 30, oracle, with_prior=False, window0=9), synth.generate_batch(3, 30, oracle, with_prior=False, window0=9)
    oracle.marginalize(cfg, src, a); gpu.marginalize(cfg, src, b)
    for w in range(3):
        A0, b0, _ = prior_canonical(a, w); A1, b1, _ = prior_canonical(b, w)
        assert np.abs(A0 - A1).max() < 1e-5 * np.abs(A0).max() and np.abs(b0 - b1).max() < 1e-4 * np.abs(b0).max()


def test_full_size_properties(gpu):
    """BASELINE.json configs[1] at full size: 1024 windows x 150 features."""
    base = synth.generate_batch(32, 150, gpu, prior_features=16, window0=2000)
    big = synth.tile_batch(base, 1024)
    st = big.state_array(); saved = big.copy_states()
    rep_a = gpu.solve_batch(big); out_a = np.frombuffer(big.states, dtype=np.uint8).copy(); lam_a = big.para_Feature.copy()
    # (1) identical inputs -> bit-identical outputs whichever CTA / wave processed them
    pose = st["para_Pose"]
    for k in range(32, 1024, 32):
        assert (pose[k:k + 32] == pose[0:32]).all()
    # (2) cost never increases and every window reports a finite result
    assert (rep_a["final_cost"] <= rep_a["initial_cost"]).all() and (rep_a["status"] == 0).all()
    assert np.abs(np.linalg.norm(pose[:, :, 3:7], axis=-1) - 1).max() < 1e-12
    # (3) the device-resident path equals the host-buffer path bit for bit
    big.restore_states(saved)
    gpu.upload(big); gpu.solve_resident(); rep_b = gpu.download(big)
    out_b = np.frombuffer(big.states, dtype=np.uint8)
    off = abi.WindowState.para_Feature.offset
    a2, b2 = out_a.reshape(1024, -1)[:, :off], out_b.reshape(1024, -1)[:, :off]
    assert (a2 == b2).all() and (lam_a == big.para_Feature).all() and (rep_a["final_cost"] == rep_b["final_cost"]).all()
    ms, launches = gpu.last_solve_stats()
    assert launches == 3 and ms > 0


def test_imu_only_windows(gpu, oracle):
    """USE_LEG == 0: IMUFactor (imu_factor.h) windows through the same kernels (EPS / RHO rows dropped, no leg bias)."""
    batch = synth.generate_batch(8, 80, gpu, use_leg=False, window0=300)
    st = batch.state_array(); lb0 = st["para_LegBias"].copy()
    rep_o, rep_g, ref, lam, st = solve_both(gpu, oracle, batch)
    assert (rep_o["iterations"] == rep_g["iterations"]).all() and (st["para_LegBias"] == lb0).all()
    d = state_diffs(st, ref)
    assert d["para_Pose"] < POS_TOL and d["para_SpeedBias"] < 1e-5, d


def test_td_open_windows(gpu, oracle):
    """ESTIMATE_TD: para_Td is the 79th camera-side unknown; it must move and match the oracle (the synthetic feature
    velocities are finite differences, so the optimum is a small window-specific offset, not exactly 0)."""
    batch = synth.generate_batch(8, 100, gpu, window0=400, prior_features=16)
    st = batch.state_array()
    for w in range(8):
        batch.descs[w].td_open = 1
    td0 = np.linspace(-0.004, 0.004, 8).reshape(8, 1); td0[np.abs(td0) < 1e-4] = 0.002
    st["para_Td"][:] = td0
    rep_o, rep_g, ref, lam, st = solve_both(gpu, oracle, batch)
    assert (rep_o["iterations"] == rep_g["iterations"]).all()
    assert np.abs(st["para_Td"] - ref["para_Td"]).max() < 1e-7
    assert (st["para_Td"] != td0).all() and np.abs(st["para_Td"]).max() < 5e-3
    d = state_diffs(st, ref)
    assert d["para_Pose"] < POS_TOL and d["para_SpeedBias"] < 1e-5 and d["para_Ex_Pose"] < POS_TOL, d


def test_maximum_feature_count(oracle):
    """NUM_OF_F = 1000 features per window (parameters.h:24, the reference's static limit): 16 chunks of tracks, 32 Schur tiles."""
    cfg = abi.default_config()
    cfg.max_batch, cfg.max_features, cfg.max_obs = 2, 1000, 1000 * 11
    big = lib.Backend(cfg)
    batch = synth.generate_batch(2, 1000, big, cfg=cfg, window0=2000, prior_features=16)
    rep_o, rep_g, ref, lam, st = solve_both(big, OracleBackend(cfg), batch, nthreads=2)
    assert (rep_o["iterations"] == rep_g["iterations"]).all()
    d = state_diffs(st, ref)
    assert d["para_Pose"] < POS_TOL and d["para_SpeedBias"] < 1e-5 and np.abs(batch.para_Feature - lam).max() < 1e-6, d


def test_rejected_steps_match_oracle_gpu():
    from test_cusim_kernels import _rejected_steps_case
    _rejected_steps_case(lambda cfg: lib.Backend(cfg))


def test_chained_windows_match_oracle_gpu():
    from test_cusim_kernels import _chained_windows_case
    _chained_windows_case(lambda cfg: lib.Backend(cfg), nw=4, F=24, F0=16, iters=8, nthreads=4)


def test_edge_windows_gpu():
    """A window without visual factors, a window with a single feature (12 iterations on the sm_90a build)."""
    from test_cusim_kernels import _empty_and_single_feature_case
    _empty_and_single_feature_case(lambda cfg: lib.Backend(cfg), iters=12)


def test_registered_host_buffers_gpu():
    """Zero-copy path with REAL page-locked memory (cudaHostRegister) and merged 2-D DMA: bit-identical to the staged path, nothing staged;
    444 windows -> 4 pipeline chunks (64, 64, 128, 188) on three compute lanes."""
    from test_cusim_kernels import _registered_buffers_case
    _registered_buffers_case(lambda cfg: lib.Backend(cfg), 512, 444, 4, iters=2)


def test_marginalization_of_imu_only_windows_gpu():
    from test_cusim_kernels import _imu_only_marginalization_case
    _imu_only_marginalization_case(lambda cfg: lib.Backend(cfg))


def test_marginalize_at_resident_solved_states(gpu, oracle):
    """cerb_batch_marginalize with states = NULL: MARGIN_OLD at the solved states as they sit on the device == the oracle's marginalization at the
    downloaded solved states."""
    cfg = abi.default_config()
    batch = synth.generate_batch(3, 40, gpu, window0=700, prior_features=12)
    gpu.solve_batch(batch)                                   # batch.states now hold the solved states, like the device
    J = np.zeros((3, abi.MAX_PRIOR_DIM * abi.MAX_PRIOR_DIM)); r = np.zeros((3, abi.MAX_PRIOR_DIM))
    priors = (abi.Prior * 3)()
    for w in range(3):
        priors[w].linearized_jacobians = J[w].ctypes.data_as(abi.c_dp); priors[w].linearized_residuals = r[w].ctypes.data_as(abi.c_dp)
    sw = gpu.batch_marginalize(np.zeros(3, dtype=np.int32), None, priors)
    assert (sw > 0).all() and (sw < 40).all()
    ref = synth.generate_batch(3, 40, gpu, window0=700, prior_features=12)
    oracle.marginalize(cfg, batch, ref)
    for w in range(3):
        A0, b0, x0 = prior_canonical(ref, w)
        n = priors[w].n
        Jm = J[w][:n * n].reshape(n, n).T
        A, g = Jm.T @ Jm, Jm.T @ r[w][:n]
        loc = {0: 6, 1: 9, 2: 4, 3: 6, 4: 1}
        keys = sorted((priors[w].block_kind[i], priors[w].block_index[i], priors[w].block_col[i]) for i in range(priors[w].num_blocks))
        perm = [c + t for (k, i, c) in keys for t in range(loc[k])]
        assert A0.shape == (n, n)
        assert np.abs(A[np.ix_(perm, perm)] - A0).max() < 1e-5 * np.abs(A0).max() and np.abs(g[perm] - b0).max() < 1e-4 * max(1.0, np.abs(b0).max())


def _shuffle_features(batch, rng):
    """Same windows, tracks handed over in a random order (the library sorts them by anchor frame on the device and returns everything in the
    caller's order).  Returns the permutation per window."""
    perms = []
    for w in range(batch.n):
        nf = batch.descs[w].n_features
        p = rng.permutation(nf)
        batch.features[w][:nf] = batch.features[w][:nf][p].copy()          # obs_offset travels with the track: the observations stay where they are
        batch.para_Feature[w][:nf] = batch.para_Feature[w][:nf][p].copy()
        perms.append(p)
    return perms


def test_full_size_feature_order_invariance(gpu):
    """Size-independent property at BASELINE.json configs[1] scale (1024 x 150): the result does not depend on the order in which the caller lists the
    tracks (device-side anchor sort, chunking, un-permutation of inverse depths / outlier errors), beyond the rounding of a different summation order."""
    base = synth.generate_batch(16, 150, gpu, realistic=True, prior_features=16, window0=2600)
    a = synth.tile_batch(base, 1024); b = synth.tile_batch(base, 1024)
    perms = _shuffle_features(b, np.random.default_rng(7))
    rep_a = gpu.solve_batch(a); err_a, _ = gpu.outlier_errors(1024)
    rep_b = gpu.solve_batch(b); err_b, _ = gpu.outlier_errors(1024)
    assert (rep_a["iterations"] == rep_b["iterations"]).all() and (rep_a["status"] == 0).all()
    assert np.abs(rep_a["final_cost"] - rep_b["final_cost"]).max() < 1e-7 * rep_a["final_cost"].max()
    d = state_diffs(a.state_array(), b.state_array())
    assert d["para_Pose"] < 1e-7 and d["para_SpeedBias"] < 1e-6 and d["para_Ex_Pose"] < 1e-7, d
    for w in range(0, 1024, 37):
        nf = a.descs[w].n_features; p = perms[w]
        assert np.abs(b.para_Feature[w][:nf] - a.para_Feature[w][:nf][p]).max() < 1e-7
        assert np.abs(err_b[w, :nf] - err_a[w, :nf][p]).max() < 1e-9


def test_gauge_covariance_of_the_solve(gpu):
    """Physics property of the whole path: without a prior the cost is invariant under a rotation about gravity + translation of the world frame, so
    solving the transformed window gives the transformed solution (the solver itself has no gauge fix: estimator.cpp:1084 pins nothing with USE_IMU)."""
    n = 8
    a = synth.generate_batch(n, 80, gpu, with_prior=False, window0=2700)
    b = synth.generate_batch(n, 80, gpu, with_prior=False, window0=2700)
    yaw, t = 0.83, np.array([3.0, -7.0, 0.4])
    Rz = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1.0]])
    qz = np.array([0, 0, np.sin(yaw / 2), np.cos(yaw / 2)])                        # (x, y, z, w)
    def qmul(p, q):      # Hamilton product, (x, y, z, w)
        px, py, pz, pw = p; qx, qy, qz_, qw = q
        return np.array([pw * qx + px * qw + py * qz_ - pz * qy, pw * qy - px * qz_ + py * qw + pz * qx, pw * qz_ + px * qy - py * qx + pz * qw, pw * qw - px * qx - py * qy - pz * qz_])
    def transform(st):
        for w in range(n):
            for i in range(11):
                st["para_Pose"][w, i, :3] = Rz @ st["para_Pose"][w, i, :3] + t
                st["para_Pose"][w, i, 3:7] = qmul(qz, st["para_Pose"][w, i, 3:7])
                st["para_SpeedBias"][w, i, :3] = Rz @ st["para_SpeedBias"][w, i, :3]
    transform(b.state_array())
    rep_a = gpu.solve_batch(a); rep_b = gpu.solve_batch(b)
    assert np.abs(rep_a["initial_cost"] - rep_b["initial_cost"]).max() < 1e-9 * rep_a["initial_cost"].max()
    assert (rep_a["iterations"] == rep_b["iterations"]).all()
    assert np.abs(rep_a["final_cost"] - rep_b["final_cost"]).max() < 1e-6 * rep_a["final_cost"].max()
    sa = a.state_array().copy(); transform(sa); sb = b.state_array()
    # the gauge itself is free (4 null directions): compare what is observable -- relative poses to frame 0, velocities, biases, depths
    for w in range(n):
        for i in range(1, 11):
            assert np.abs((sa["para_Pose"][w, i, :3] - sa["para_Pose"][w, 0, :3]) - (sb["para_Pose"][w, i, :3] - sb["para_Pose"][w, 0, :3])).max() < 2e-4
    assert np.abs(sa["para_SpeedBias"][:, :, 3:] - sb["para_SpeedBias"][:, :, 3:]).max() < 1e-4 and np.abs(sa["para_LegBias"] - sb["para_LegBias"]).max() < 1e-6
    assert np.abs(a.para_Feature - b.para_Feature).max() < 1e-4
