"""Per-feature steps either side of the solve (SURVEY.md 8(f) n3): Estimator::outliersRejection and FeatureManager::triangulate
on the resident batch.  CPU tier: the kernels on the CPU simulator vs the oracle restatement (estimator.cpp:1729-1798,
feature_manager.cpp:198-212,302-385), the oracle's 4x4 null vector vs numpy's LAPACK SVD, and the geometry itself (a noise-free
track triangulates to its true depth).  GPU tier: the sm_90a kernels vs the oracle."""
import numpy as np
import pytest
from cerberus_b200 import abi, synth
from oracle_lib import OracleBackend
from helpers import sim_backend, small_cfg


def _batch(backend, realistic, n=2, F=24):
    batch = synth.generate_batch(n, F, backend, realistic=realistic, window0=77, prior_features=8)
    for w in range(n):                                           # one two-frame track anchored at frame 0 per window: removeBackShiftDepth erases it
        f = next(f for f in range(batch.descs[w].n_features) if batch.descs[w].features[f].start_frame == 0)
        batch.descs[w].features[f].n_obs = 2
    return batch


def _check_backend(be, oracle, realistic):
    batch = _batch(be, realistic)
    nf = [batch.descs[w].n_features for w in range(batch.n)]
    # (1) outlier errors at the initial states and after the solve
    be.upload(batch)
    for phase in range(2):
        err, rem = be.outlier_errors(batch.n)
        ref = oracle.outlier_errors(batch)
        for w in range(batch.n):
            ok = np.isfinite(ref[w, :nf[w]])     # the reference's own loop skips tracks with used_num < 4 (estimator.cpp:1750); the ABI never passes them to a solve
            assert ok.sum() >= nf[w] - 1
            assert np.abs(err[w, :nf[w]][ok] - ref[w, :nf[w]][ok]).max() < 1e-12 * max(1.0, np.abs(ref[w, :nf[w]][ok]).max())
            assert (rem[w, :nf[w]][ok] == (ref[w, :nf[w]][ok] * 460.0 > 3)).all()
        if phase == 0:
            be.solve_resident(); be.download(batch)           # batch.states now hold the solved states, like the device
    assert np.nanmax(err) * 460.0 < 3.0                           # solved synthetic windows have no outliers
    # (1a) cerb_batch_update_states: the window moved (double2vector + vector2double), only the states travel; same as a full upload of the moved window
    rng = np.random.default_rng(3)
    st = batch.state_array()
    st["para_Pose"][:, :, :3] += rng.normal(0, 0.01, st["para_Pose"][:, :, :3].shape)
    for w in range(batch.n): batch.para_Feature[w, :nf[w]] *= 1.0 + rng.normal(0, 0.01, nf[w])
    be.update_states(batch); err_u, rem_u = be.outlier_errors(batch.n)
    be.upload(batch); err_f, rem_f = be.outlier_errors(batch.n)
    ref = oracle.outlier_errors(batch)
    for w in range(batch.n):
        ok = np.isfinite(ref[w, :nf[w]])
        assert (err_u[w, :nf[w]] == err_f[w, :nf[w]]).all() and (rem_u[w] == rem_f[w]).all()
        assert np.abs(err_u[w, :nf[w]][ok] - ref[w, :nf[w]][ok]).max() < 1e-12 * max(1.0, np.abs(ref[w, :nf[w]][ok]).max())
    # (1a') a resident solve after the update starts from the shipped states: same result as solving the moved window from host buffers
    import copy
    moved = synth.tile_batch(batch, batch.n)                        # deep copy (descriptors + states)
    be.update_states(batch); be.solve_resident(); rep_r = be.download(batch)
    rep_h = be.solve_batch(moved)
    assert (rep_r["iterations"] == rep_h["iterations"]).all() and np.abs(rep_r["final_cost"] - rep_h["final_cost"]).max() < 1e-9 * np.abs(rep_h["final_cost"]).max()
    assert np.abs(batch.state_array()["para_Pose"] - moved.state_array()["para_Pose"]).max() < 1e-10
    be.upload(batch)                                                 # the solved states again, for the passes below
    # (1b) depth bookkeeping of slideWindowOld at the solved states
    st_o, dep_o, keep_o = oracle.shift_depth(batch)
    st_g, dep_g, keep_g = be.shift_depth(batch.n)
    for w in range(batch.n):
        kp = keep_o[w, :nf[w]] != 0                 # erased tracks have no start frame / depth in the reference (the list node is gone)
        assert (keep_g[w, :nf[w]] == keep_o[w, :nf[w]]).all() and (st_g[w, :nf[w]][kp] == st_o[w, :nf[w]][kp]).all()
        assert np.abs(dep_g[w, :nf[w]][kp] - dep_o[w, :nf[w]][kp]).max() < 1e-12 * np.abs(dep_o[w, :nf[w]][kp]).max()
        assert (dep_g[w, :nf[w]] > 0).all() and (keep_o[w, :nf[w]] == 0).sum() == 1 and (st_o[w, :nf[w]][kp] >= 0).all()
    # (2) triangulation: mark every second feature as not triangulated (estimated_depth = -1 -> para_Feature = -1)
    true_depth = 1.0 / batch.para_Feature.copy()
    for w in range(batch.n):
        batch.para_Feature[w, 0:nf[w]:2] = -1.0
    be.upload(batch)
    st_o, dep_o, keep_o = oracle.shift_depth(batch, 7.5); st_g, dep_g, keep_g = be.shift_depth(batch.n, 7.5)    # negative depths -> INIT_DEPTH
    for w in range(batch.n):
        kp = keep_o[w, :nf[w]] != 0
        assert (dep_g[w, :nf[w]][kp] == dep_o[w, :nf[w]][kp]).all() or np.abs(dep_g[w, :nf[w]][kp] - dep_o[w, :nf[w]][kp]).max() < 1e-12 * 20
    assert realistic or (dep_o == 7.5).any()
    dep = be.triangulate(batch.n)
    ref = oracle.triangulate(batch)
    for w in range(batch.n):
        assert np.abs(dep[w, :nf[w]] - ref[w, :nf[w]]).max() < 1e-8 * np.abs(ref[w, :nf[w]]).max()
        assert (dep[w, 1:nf[w]:2] == 1.0 / batch.para_Feature[w, 1:nf[w]:2]).all()          # untouched features: current depth
        # sanity of the geometry: positive depths of the right magnitude (a 0.5-px-noise stereo pair with a ~0.1 m baseline only
        # constrains depths of 2..15 m to a few tens of percent)
        assert (dep[w, 0:nf[w]:2] > 0).all() and np.median(np.abs(dep[w, 0:nf[w]:2] / true_depth[w, 0:nf[w]:2] - 1.0)) < 0.6


@pytest.mark.parametrize("realistic", [False, True])
def test_feature_steps_sim(realistic):
    cfg = small_cfg(max_batch=4, max_features=24, iters=3)
    _check_backend(sim_backend(cfg), OracleBackend(cfg), realistic)


def test_oracle_null_vector_vs_lapack():
    """The oracle's triangulation on exact two-view geometry: numpy (LAPACK) SVD of the same design matrix gives the same point."""
    rng = np.random.default_rng(5)
    for _ in range(20):
        X = np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), rng.uniform(3, 12)])
        t1 = np.array([0.2, rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05)])
        P0 = np.hstack([np.eye(3), np.zeros((3, 1))]); P1 = np.hstack([np.eye(3), -t1[:, None]])
        u0 = X[:2] / X[2]; x1 = X - t1; u1 = x1[:2] / x1[2]
        A = np.stack([u0[0] * P0[2] - P0[0], u0[1] * P0[2] - P0[1], u1[0] * P1[2] - P1[0], u1[1] * P1[2] - P1[1]])
        v = np.linalg.svd(A)[2][-1]
        assert np.abs(v[:3] / v[3] - X).max() < 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("realistic", [False, True])
def test_feature_steps_gpu(realistic):
    from cerberus_b200 import lib
    cfg = small_cfg(max_batch=4, max_features=24, iters=4)
    _check_backend(lib.Backend(cfg), OracleBackend(cfg), realistic)
