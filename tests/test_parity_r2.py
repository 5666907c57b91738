"""Parity holes named by the round-1 review, closed (both tiers).

CPU tier (`-m "not gpu"`):
  * cerb_double2vector (the gauge re-anchoring of Estimator::double2vector, estimator.cpp:903-957 -- the function that produces the
    poses the estimator publishes) against the oracle restatement AND against the reference's own Utility::R2ypr / ypr2R
    (utils/utility.cpp compiled into oracle/_ref), including the singular-pitch branch (:925-934);
  * the per-feature steps (triangulate / outlier errors / depth shift) of the oracle and of the kernels (CPU simulator) against
    the reference's own FeatureManager (featureTracker/feature_manager.cpp compiled into oracle/_ref) and the statements of
    Estimator::reprojectionError / outliersRejection executed over it.
The reference arm replays the stored outputs of those sources (tests/golden/ref_v1.npz, see tests/oracle_lib.py).
GPU tier (`-m gpu`): the sm_90a build of cerb_preintegrate_imu_batch, cerb_eval_imu, cerb_eval_prior, the sum_dt > 10 skipped
factor, MARGIN_SECOND_NEW and marginalization with an old prior, the per-feature steps against the reference sources."""
import ctypes as C
import os
import numpy as np
import pytest
from cerberus_b200 import abi, synth, lib
from oracle_lib import OracleBackend, RefBackend, ref_rows, sub_jobs
from helpers import sim_backend, small_cfg, prior_canonical, state_diffs, SIM_LIB
from test_preintegration import make_jobs

ob = OracleBackend()


# ---------------------------------------------------------------------------------------------------- double2vector
def _Rz(a): return np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
def _Ry(a): return np.array([[np.cos(a), 0, np.sin(a)], [0, 1.0, 0], [-np.sin(a), 0, np.cos(a)]])
def _Rx(a): return np.array([[1.0, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])


def _quat(R):
    from cerberus_b200.estimator import R_to_quat
    return R_to_quat(R)


def _d2v_states(rng, pitch_before_deg, pitch_after_deg):
    """(before, after): frame 0 of `before` / `after` have the given pitch; everything else random."""
    before, after = abi.WindowState(), abi.WindowState()
    for st, pitch in ((before, pitch_before_deg), (after, pitch_after_deg)):
        for i in range(abi.NUM_FRAMES):
            y, r = rng.uniform(-np.pi, np.pi), rng.uniform(-0.5, 0.5)
            p = np.deg2rad(pitch) if i == 0 else rng.uniform(-0.6, 0.6)
            q = _quat(_Rz(y) @ _Ry(p) @ _Rx(r)) * (1.0 + (rng.uniform(-1e-9, 1e-9) if st is after else 0.0))   # after: not exactly unit (normalized() matters)
            if rng.uniform() < 0.3: q = -q
            st.para_Pose[i][0:3] = list(rng.normal(0, 3, 3)); st.para_Pose[i][3:7] = list(q)
            st.para_SpeedBias[i][0:9] = list(rng.normal(0, 1, 9))
    return before, after


def _d2v_product(cdll, before, after):
    Ps, Rs, Vs = np.zeros((11, 3)), np.zeros((11, 3, 3)), np.zeros((11, 3))
    cdll.cerb_double2vector.restype = None
    cdll.cerb_double2vector.argtypes = [C.POINTER(abi.WindowState), C.POINTER(abi.WindowState), abi.c_dp, abi.c_dp, abi.c_dp]
    cdll.cerb_double2vector(C.byref(before), C.byref(after), Ps.ctypes.data_as(abi.c_dp), Rs.ctypes.data_as(abi.c_dp), Vs.ctypes.data_as(abi.c_dp))
    return Ps, Rs, Vs


D2V_PITCHES = [(5.0, -7.0), (30.0, 29.0), (-45.0, -44.0), (89.6, 20.0), (10.0, -89.3), (-89.9, -89.9), (88.9, 88.9), (91.0 - 2.0, 40.0)]


def _check_d2v(cdll):
    rng = np.random.default_rng(12)
    ref = RefBackend()
    singular = 0
    for k, (pb, pa) in enumerate(D2V_PITCHES * 3):
        before, after = _d2v_states(rng, pb, pa)
        got = _d2v_product(cdll, before, after)
        for arm in ((ob, ref) if k < len(D2V_PITCHES) else (ob,)):      # the reference arm on the first pass over the pitches
            want = arm.double2vector(before, after)
            for g, w, name in zip(got, want, ("Ps", "Rs", "Vs")):
                assert np.abs(g - w).max() < 1e-12 * max(1.0, np.abs(w).max()), (name, pb, pa, type(arm).__name__)
        # the property the step exists for: frame 0 keeps its position and its yaw
        assert np.abs(got[0][0] - np.array(before.para_Pose[0][0:3])).max() < 1e-12
        if abs(abs(pb) - 90) < 1.0 or abs(abs(pa) - 90) < 1.0:
            singular += 1
            from cerberus_b200.estimator import quat_to_R
            assert np.abs(got[1][0] - quat_to_R(np.array(before.para_Pose[0][3:7]))).max() < 1e-7      # rot_diff = Rs0 R00^T (R00 from the un-normalised quaternion, as in the reference)
    assert singular >= 9


def test_double2vector_sim_build_vs_oracle_and_reference():
    _check_d2v(C.CDLL(SIM_LIB) if os.path.exists(SIM_LIB) else sim_backend(small_cfg()).lib)


def test_double2vector_product_library_vs_oracle_and_reference():
    """The sm_90a library's host-side cerb_double2vector (no device involved: callable without a GPU)."""
    if not os.path.exists(lib.PRODUCT_LIB):
        pytest.skip("product library not built")
    try:
        cdll = C.CDLL(lib.PRODUCT_LIB)
    except OSError as e:       # libcudart missing on this machine
        pytest.skip(str(e))
    _check_d2v(cdll)


# ---------------------------------------------------------------------------------------------------- n3 against reference source
@pytest.mark.parametrize("realistic", [False, True])
def test_feature_steps_oracle_and_sim_vs_reference_feature_manager(realistic):
    """FeatureManager::{triangulate, triangulatePoint, removeBackShiftDepth} (feature_manager.cpp:198-212,302-385,450-488) and the
    statements of Estimator::{reprojectionError, outliersRejection} (estimator.cpp:1729-1798) executed from the reference's source,
    against the oracle restatement and the kernels (CPU simulator).  The kernels along a solve are checked against the oracle by
    test_feature_steps.py."""
    cfg = small_cfg(max_batch=4, max_features=24, iters=3)
    _check_feature_steps_vs_reference(ob, realistic)
    _check_feature_steps_vs_reference(sim_backend(cfg), realistic)


def _feature_steps(arm, batch):
    """(outlier errors, triangulated depths, (start frame, depth, keep) of the depth shift) of `arm` at the batch's states: the
    oracle and the reference read the host batch, a library backend gets it uploaded before each step."""
    if not isinstance(arm, lib.Backend):
        return arm.outlier_errors(batch), arm.triangulate(batch), arm.shift_depth(batch, 6.5)
    arm.upload(batch); e = arm.outlier_errors(batch.n)[0]
    arm.upload(batch); t = arm.triangulate(batch.n)
    arm.upload(batch); s = arm.shift_depth(batch.n, 6.5)
    return e, t, s


def _check_feature_steps_vs_reference(arm, realistic):
    """The per-feature steps of `arm` against the reference's FeatureManager on the windows of test_feature_steps._batch (built by the
    oracle, so the inputs do not depend on the arm), once as generated and once with every second track not triangulated."""
    from test_feature_steps import _batch
    ref = RefBackend()
    batch = _batch(ob, realistic)
    nf = [batch.descs[w].n_features for w in range(batch.n)]
    for lamset in (0, 1):
        if lamset:
            for w in range(batch.n):
                batch.para_Feature[w, 0:nf[w]:2] = -1.0
        (e0, t0, s0), (e1, t1, s1) = _feature_steps(arm, batch), _feature_steps(ref, batch)
        for w in range(batch.n):
            k = nf[w]
            if not lamset:
                ok = np.isfinite(e1[w, :k])         # the reference skips used_num < 4 (estimator.cpp:1750)
                assert ok.sum() >= k - 1 and np.abs(e0[w, :k][ok] - e1[w, :k][ok]).max() < 1e-12 * max(1.0, np.abs(e1[w, :k][ok]).max())
            assert np.abs(t0[w, :k] - t1[w, :k]).max() < 1e-8 * np.abs(t1[w, :k]).max()
            keep = s1[2][w, :k] != 0
            assert (s0[0][w, :k][keep] == s1[0][w, :k][keep]).all() and (s0[2][w, :k] == s1[2][w, :k]).all()
            assert np.abs(s0[1][w, :k][keep] - s1[1][w, :k][keep]).max() < 1e-12 * np.abs(s1[1][w, :k][keep]).max()


# ---------------------------------------------------------------------------------------------------- GPU tier
def _gpu(cfg=None):
    return lib.Backend(cfg or small_cfg(max_batch=8, max_features=32))


@pytest.mark.gpu
def test_double2vector_product_library_gpu_box():
    _check_d2v(_gpu().lib)


@pytest.mark.gpu
def test_imu_preintegration_and_imu_factor_gpu():
    """Row a9 / a6 on the sm_90a build: cerb_preintegrate_imu_batch and cerb_eval_imu vs the oracle and the reference's
    integration_base.h / imu_factor.h (oracle/_ref)."""
    from test_reference_pin import imu_setup
    gpu = _gpu()
    ref = RefBackend()
    jobs, _, _ = make_jobs(6, seed=29)
    pcfg = abi.default_preint_config()
    got = gpu.preintegrate_imu(pcfg, jobs, 6)
    rows = ref_rows(6, 2)
    for arm, want, sel in ((ob, ob.preintegrate_imu(pcfg, jobs, 6), slice(None)), (ref, ref.preintegrate_imu(pcfg, sub_jobs(jobs, rows), len(rows)), rows)):
        for name in want.dtype.names:
            assert np.abs(got[sel][name] - want[name]).max() <= 1e-11 * max(1e-30, np.abs(want[name]).max()), (name, type(arm).__name__)
    pre, params = imu_setup(4)
    rows = ref_rows(4, 1)
    out = gpu.eval_imu(pre, params)
    for arm, (r0, j0, s0), sel in ((ob, ob.eval_imu(pre, params), slice(None)), (ref, ref.eval_imu(pre[rows], params[rows]), rows)):
        r1, j1, s1 = (x[sel] for x in out)
        assert np.abs(s0 - s1).max() < 1e-9 * np.abs(s0).max() and np.abs(r0 - r1).max() < 1e-9 * np.abs(r0).max() and np.abs(j0 - j1).max() < 1e-9 * np.abs(j0).max()
    # the windows a USE_LEG == 0 estimator would solve, fed by the DEVICE preintegration on one arm and the oracle's on the other
    cfg = small_cfg(max_batch=4, max_features=32)
    g2, o2 = lib.Backend(cfg), OracleBackend(cfg)
    bg = synth.generate_batch(2, 24, g2, use_leg=False, window0=310)
    bo = synth.generate_batch(2, 24, o2, use_leg=False, window0=310)
    for name in bo.imu_preint.dtype.names:
        assert np.abs(bg.imu_preint[name] - bo.imu_preint[name]).max() <= 1e-11 * max(1e-30, np.abs(bo.imu_preint[name]).max()), name
    rep_g = g2.solve_batch(bg); rep_o = o2.solve_batch(bo)
    assert (rep_g["iterations"] == rep_o["iterations"]).all()
    assert state_diffs(bg.state_array(), bo.state_array())["para_Pose"] < 1e-6


@pytest.mark.gpu
def test_prior_evaluator_gpu():
    """cerb_eval_prior (MarginalizationFactor::Evaluate, marginalization_factor.cpp:347-395) on the device vs oracle and reference."""
    gpu = _gpu()
    batch = synth.generate_batch(1, 8, ob, prior_features=6)
    st = batch.state_array()
    st["para_Pose"][0, :, :3] += 0.02; st["para_SpeedBias"][0, 0] += 0.01; st["para_LegBias"][0, 0] += 1e-3
    st["para_Pose"][0, :, 3:7] += 0.003; st["para_Pose"][0, :, 3:7] /= np.linalg.norm(st["para_Pose"][0, :, 3:7], axis=-1, keepdims=True)
    st["para_Pose"][0, 2, 3:7] *= -1.0                       # w < 0 branch of the rotation residual (:369-375)
    pr = batch.descs[0].prior
    ncols = 7 * 12 + 9 + 4 + 1
    r1, j1 = gpu.eval_prior(pr, batch.states[0], ncols)
    rows = ref_rows(pr.n, 12)
    r2, j2 = ob.eval_prior(pr, batch.states[0], ncols)
    for (r0, j0), sel in (((r2, j2.reshape(pr.n, ncols)), slice(None)), (RefBackend().eval_prior(pr, batch.states[0], ncols, rows), rows)):
        r1s, j1s = r1[sel], j1.reshape(pr.n, ncols)[sel]
        assert np.abs(r0 - r1s).max() < 1e-10 * np.abs(r0).max() and np.abs(j0 - j1s).max() == 0.0


@pytest.mark.gpu
def test_skipped_imu_factor_gpu():
    """estimator.cpp:1119 (sum_dt > 10: factor not added) on the sm_90a build."""
    cfg = small_cfg(max_batch=4, max_features=32, iters=6)
    o, g = OracleBackend(cfg), lib.Backend(cfg)
    batch = synth.generate_batch(3, 24, o, window0=31, prior_features=8)
    batch.preint[0][3]["sum_dt"] = 10.5
    batch.preint[1][0]["sum_dt"] = 12.0; batch.preint[1][9]["sum_dt"] = 11.0
    st = batch.state_array(); saved = batch.copy_states()
    rep_o = o.solve_batch(batch); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_g = g.solve_batch(batch)
    assert (rep_o["iterations"] == rep_g["iterations"]).all() and (rep_o["num_successful_steps"] == rep_g["num_successful_steps"]).all()
    assert np.abs(rep_o["final_cost"] - rep_g["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    d = state_diffs(batch.state_array(), ref)
    assert d["para_Pose"] < 1e-6 and d["para_SpeedBias"] < 1e-5 and np.abs(batch.para_Feature - lam).max() < 1e-6, d


@pytest.mark.gpu
@pytest.mark.parametrize("margin_old", [True, False])
def test_marginalization_with_prior_gpu(margin_old):
    """MARGIN_OLD with an existing prior and MARGIN_SECOND_NEW on the sm_90a build vs the reference's MarginalizationInfo classes and the oracle."""
    cfg = small_cfg()
    gpu = lib.Backend(cfg)
    mk = lambda: synth.generate_batch(2, 10, ob, with_prior=True, window0=47)
    src = mk()
    c = mk(); gpu.marginalize(cfg, src, c, margin_old)
    a = mk(); ob.marginalize(cfg, src, a, margin_old)
    for want in ([prior_canonical(a, w) for w in range(2)], RefBackend().marginal_priors(cfg, synth.tile_batch(src, 1), margin_old)):
        for w in range(len(want)):
            (A0, b0, x0), (A1, b1, x1) = want[w], prior_canonical(c, w)
            assert A0.shape[0] == (86 if margin_old else 80) and A0.shape == A1.shape and set(x0) == set(x1)
            assert np.abs(A0 - A1).max() < 1e-5 * np.abs(A0).max() and np.abs(b0 - b1).max() < 1e-4 * np.abs(b0).max()
            assert all(np.abs(x0[k][:7] - x1[k][:7]).max() == 0 for k in x0)


@pytest.mark.gpu
@pytest.mark.parametrize("realistic", [False, True])
def test_feature_steps_gpu_vs_reference_feature_manager(realistic):
    _check_feature_steps_vs_reference(lib.Backend(small_cfg(max_batch=4, max_features=24, iters=4)), realistic)


@pytest.mark.gpu
def test_stress_feature_count_gpu():
    """BASELINE.json configs[4]: 10-frame x 2000-feature windows (dense Schur: 32 chunks of tracks, 63 Schur tiles, the inverse-depth scales in the
    global workspace instead of shared memory).  Exceeds the reference's static NUM_OF_F = 1000 (parameters.h:24) on purpose; parity vs the oracle."""
    cfg = abi.default_config()
    cfg.max_batch, cfg.max_features, cfg.max_obs = 2, 2000, 2000 * 11
    big = lib.Backend(cfg)
    o = OracleBackend(cfg)
    batch = synth.generate_batch(2, 2000, big, cfg=cfg, window0=4000, prior_features=16)
    st = batch.state_array(); saved = batch.copy_states()
    rep_o = o.solve_batch(batch, nthreads=2); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_g = big.solve_batch(batch)
    assert (rep_o["iterations"] == rep_g["iterations"]).all() and (rep_o["num_successful_steps"] == rep_g["num_successful_steps"]).all()
    d = state_diffs(batch.state_array(), ref)
    assert d["para_Pose"] < 1e-6 and d["para_SpeedBias"] < 1e-5 and np.abs(batch.para_Feature - lam).max() < 1e-6, d
    # over the capacity limit of the library
    cfg2 = abi.default_config(); cfg2.max_batch, cfg2.max_features, cfg2.max_obs = 1, 2049, 2049 * 11
    with pytest.raises(lib.CerbError):
        lib.Backend(cfg2)
