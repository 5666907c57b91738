"""The sm_90a kernel sources, run on CPU threads by tests/cusim, against the CPU oracle (non-GPU tier).
The same comparisons run on the real device in test_gpu_parity.py."""
import numpy as np
import pytest
from cerberus_b200 import abi, synth
from oracle_lib import OracleBackend
from helpers import sim_backend, small_cfg, state_diffs, prior_canonical
from test_oracle_jacobians import proj_inputs, imu_leg_setup

ob = OracleBackend()


@pytest.fixture(scope="module")
def sb():
    return sim_backend(small_cfg())


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_projection_kernel(sb, kind):
    args = proj_inputs(np.random.default_rng(kind), 40)
    r0, j0 = ob.eval_projection(kind, *args)
    r1, j1 = sb.eval_projection(kind, *args)
    assert np.abs(r0 - r1).max() < 1e-9 * max(1.0, np.abs(r0).max())
    assert np.abs(j0 - j1).max() < 1e-10 * np.abs(j0).max()


def test_imu_leg_kernel(sb):
    pre, params = imu_leg_setup(3)
    r0, j0, s0 = ob.eval_imu_leg(pre, params)
    r1, j1, s1 = sb.eval_imu_leg(pre, params)
    assert np.abs(s0 - s1).max() < 1e-10 * np.abs(s0).max()
    assert np.abs(r0 - r1).max() < 1e-9 * np.abs(r0).max()
    assert np.abs(j0 - j1).max() < 1e-9 * np.abs(j0).max()


def test_prior_kernel(sb):
    batch = synth.generate_batch(1, 8, ob, prior_features=6)
    st = batch.state_array()
    st["para_Pose"][0, :, :3] += 0.01; st["para_Pose"][0, :, 3:7] += 0.002
    st["para_Pose"][0, :, 3:7] /= np.linalg.norm(st["para_Pose"][0, :, 3:7], axis=-1, keepdims=True)
    st["para_SpeedBias"][0, 0] += 0.01
    pr = batch.descs[0].prior
    ncols = 7 * 12 + 9 + 4 + 1
    r0, j0 = ob.eval_prior(pr, batch.states[0], ncols)
    r1, j1 = sb.eval_prior(pr, batch.states[0], ncols)
    assert np.abs(r0 - r1).max() < 1e-9 * np.abs(r0).max() and np.abs(j0 - j1).max() == 0.0


@pytest.mark.parametrize("realistic,iters", [(False, 3), (True, 4)])
def test_fused_solve_matches_oracle(realistic, iters):
    cfg = small_cfg(iters=iters)
    o, s = OracleBackend(cfg), sim_backend(cfg)
    batch = synth.generate_batch(2, 10, o, realistic=realistic, window0=11, prior_features=6)
    st = batch.state_array(); saved = batch.copy_states()
    # linearisation probe: cost, gradient and diag(J^T J) at the initial point
    s.upload(batch)
    cost, g, d = s.debug_linearize(batch, 1)
    g0, d0 = o.solve_window(batch, 1, want_probe=True)
    assert abs(cost - batch.reports[1].initial_cost) < 1e-9 * cost
    assert np.abs(g - g0).max() < 1e-9 * np.abs(g0).max()
    assert (np.abs(d - d0) / np.maximum(np.abs(d0), 1e-300)).max() < 1e-8
    batch.restore_states(saved)
    rep_o = o.solve_batch(batch); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_s = s.solve_batch(batch)
    assert (rep_o["iterations"] == rep_s["iterations"]).all() and (rep_o["num_successful_steps"] == rep_s["num_successful_steps"]).all()
    assert np.abs(rep_o["final_cost"] - rep_s["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    diffs = state_diffs(batch.state_array(), ref)
    assert diffs["para_Pose"] < 1e-7 and diffs["para_SpeedBias"] < 1e-6 and diffs["para_Ex_Pose"] < 1e-7, diffs
    assert np.abs(batch.para_Feature - lam).max() < 1e-7


def test_masked_blocks_and_missing_prior():
    """ex / leg bias constant, no prior: the masked dimensions must not move and the rest must match the oracle."""
    cfg = small_cfg(iters=3); cfg.optimize_leg_bias = 0
    o, s = OracleBackend(cfg), sim_backend(cfg)
    batch = synth.generate_batch(1, 10, o, with_prior=False, window0=3)
    batch.descs[0].extrinsic_open = 0
    st = batch.state_array(); saved = batch.copy_states()
    ex0, lb0 = st["para_Ex_Pose"].copy(), st["para_LegBias"].copy()
    o.solve_batch(batch); ref = st.copy()
    batch.restore_states(saved)
    s.solve_batch(batch)
    st = batch.state_array()
    assert (st["para_Ex_Pose"] == ex0).all() and (st["para_LegBias"] == lb0).all()
    assert state_diffs(st, ref)["para_Pose"] < 1e-7


def test_marginalization_glue_matches_oracle(sb):
    """MARGIN_OLD through the device evaluators + numpy glue vs the oracle's restatement: same information matrix."""
    cfg = small_cfg()
    for realistic in (False, True):
        src = synth.generate_batch(2, 10, ob, realistic=realistic, with_prior=False, window0=21)
        if realistic:
            src.features[:, :4]["start_frame"] = 0       # make sure some features are anchored at frame 0
            src.features[:, :4]["n_obs"] = np.minimum(src.features[:, :4]["n_obs"], 11)
        a, b = synth.generate_batch(2, 10, ob, with_prior=False, window0=21), synth.generate_batch(2, 10, ob, with_prior=False, window0=21)
        ob.marginalize(cfg, src, a); sb.marginalize(cfg, src, b)
        for w in range(2):
            A0, b0, x0 = prior_canonical(a, w); A1, b1, x1 = prior_canonical(b, w)
            assert A0.shape == A1.shape
            assert np.abs(A0 - A1).max() < 1e-5 * np.abs(A0).max() and np.abs(b0 - b1).max() < 1e-4 * np.abs(b0).max()
            assert all(np.abs(x0[k] - x1[k]).max() == 0 for k in x0)


def test_imu_only_window_solve():
    """USE_LEG == 0 (estimator.cpp:1160-1171): IMUFactor windows, no leg-bias blocks, no prior."""
    cfg = small_cfg(iters=3)
    o, s = OracleBackend(cfg), sim_backend(cfg)
    batch = synth.generate_batch(1, 10, o, use_leg=False, window0=55)
    st = batch.state_array(); saved = batch.copy_states(); lb0 = st["para_LegBias"].copy()
    rep_o = o.solve_batch(batch); ref = st.copy()
    batch.restore_states(saved)
    rep_s = s.solve_batch(batch)
    st = batch.state_array()
    assert (rep_o["iterations"] == rep_s["iterations"]).all() and (st["para_LegBias"] == lb0).all()
    assert abs(rep_o["final_cost"][0] - rep_s["final_cost"][0]) < 1e-7 * rep_o["final_cost"][0]
    d = state_diffs(st, ref)
    assert d["para_Pose"] < 1e-7 and d["para_SpeedBias"] < 1e-6, d


def test_td_open_window_solve():
    """ESTIMATE_TD (estimator.cpp:1114-1123 adds para_Td unless it is held constant): td is the 79th camera-side
    unknown; gradient/diagonal probe, iteration counts, the td estimate and the poses must match the oracle."""
    cfg = small_cfg(iters=4)
    o, s = OracleBackend(cfg), sim_backend(cfg)
    batch = synth.generate_batch(2, 12, o, window0=77, prior_features=6)
    st = batch.state_array()
    for w in range(2):
        batch.descs[w].td_open = 1
    st["para_Td"][:, 0] = [0.004, -0.003]
    saved = batch.copy_states()
    s.upload(batch)
    cost, g, d = s.debug_linearize(batch, 0)
    g0, d0 = o.solve_window(batch, 0, want_probe=True)
    assert g0[221] != 0.0 and d0[221] > 0.0
    assert np.abs(g - g0).max() < 1e-9 * np.abs(g0).max()
    assert (np.abs(d - d0) / np.maximum(np.abs(d0), 1e-300)).max() < 1e-8
    batch.restore_states(saved)
    rep_o = o.solve_batch(batch); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_s = s.solve_batch(batch)
    st = batch.state_array()
    assert (rep_o["iterations"] == rep_s["iterations"]).all() and (rep_o["num_successful_steps"] == rep_s["num_successful_steps"]).all()
    assert np.abs(rep_o["final_cost"] - rep_s["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    assert (st["para_Td"] != saved_td(saved)).all()
    assert np.abs(st["para_Td"] - ref["para_Td"]).max() < 1e-8
    diffs = state_diffs(st, ref)
    assert diffs["para_Pose"] < 1e-7 and diffs["para_SpeedBias"] < 1e-6 and diffs["para_Ex_Pose"] < 1e-7, diffs
    assert np.abs(batch.para_Feature - lam).max() < 1e-7


def saved_td(saved):
    return np.array([[0.004], [-0.003]])


def test_empty_and_single_feature_windows():
    _empty_and_single_feature_case(sim_backend)


def _empty_and_single_feature_case(make_backend, iters=3):
    """Edge cases of the track list: a window with no visual factors at all (IMU-leg factors + prior only) and one with a
    single feature; both must match the oracle."""
    cfg = small_cfg(max_batch=2, max_features=16, iters=iters)
    o, s = OracleBackend(cfg), make_backend(cfg)
    batch = synth.generate_batch(2, 10, o, window0=5, prior_features=6)
    batch.descs[0].n_features = 0; batch.descs[0].n_obs = 0
    batch.descs[1].n_features = 1
    st = batch.state_array(); saved = batch.copy_states()
    rep_o = o.solve_batch(batch); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_s = s.solve_batch(batch)
    assert (rep_o["iterations"] == rep_s["iterations"]).all()
    assert np.abs(rep_o["final_cost"] - rep_s["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    d = state_diffs(batch.state_array(), ref)
    assert d["para_Pose"] < 1e-7 and d["para_SpeedBias"] < 1e-6 and np.abs(batch.para_Feature - lam).max() < 1e-7


def _rejected_steps_case(backend_factory, nw=6, iters=12):
    """Windows whose trust region rejects steps (min_relative_decrease raised to 0.97 for both sides): exercises the dogleg re-use
    path after a rejected step -- in particular after a rejected SPECULATIVE linearisation of the candidate -- against the oracle."""
    cfg = small_cfg(max_batch=6, max_features=16, iters=iters)
    cfg.min_relative_decrease = 0.97
    o, s = OracleBackend(cfg), backend_factory(cfg)
    batch = synth.generate_batch(nw, 12, o, window0=900 + (6 - nw), prior_features=6)
    st = batch.state_array()
    rng = np.random.default_rng(3)
    for w in range(nw):
        st["para_Pose"][w, :, :3] += rng.normal(0, 0.1 + 0.1 * w, (11, 3))
        batch.para_Feature[w] *= np.exp(rng.normal(0, 0.5, batch.para_Feature.shape[1]))
    saved = batch.copy_states()
    rep_o = o.solve_batch(batch); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_s = s.solve_batch(batch)
    assert (rep_o["num_successful_steps"] < rep_o["iterations"]).any()          # the case does contain rejected steps
    assert (rep_o["iterations"] == rep_s["iterations"]).all() and (rep_o["num_successful_steps"] == rep_s["num_successful_steps"]).all()
    assert np.abs(rep_o["final_cost"] - rep_s["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    d = state_diffs(batch.state_array(), ref)
    assert d["para_Pose"] < 1e-6 and d["para_SpeedBias"] < 1e-6 and np.abs(batch.para_Feature - lam).max() < 1e-6, d


def test_rejected_steps_match_oracle():
    _rejected_steps_case(sim_backend, nw=3, iters=9)          # (the GPU tier runs the 6-window / 12-iteration case)


def test_skipped_imu_factor():
    """estimator.cpp:1119: an IMU-leg factor whose sum_dt exceeds 10 s is not added; the frames it would couple are then tied
    together by the visual factors and the prior only."""
    cfg = small_cfg(max_batch=2, max_features=16, iters=3)
    o, s = OracleBackend(cfg), sim_backend(cfg)
    batch = synth.generate_batch(2, 12, o, window0=31, prior_features=6)
    batch.preint[0][3]["sum_dt"] = 10.5          # window 0: factor 3 skipped
    batch.preint[1][0]["sum_dt"] = 12.0          # window 1: factors 0 and 9 skipped
    batch.preint[1][9]["sum_dt"] = 11.0
    st = batch.state_array(); saved = batch.copy_states()
    rep_o = o.solve_batch(batch); ref = st.copy(); lam = batch.para_Feature.copy()
    batch.restore_states(saved)
    rep_s = s.solve_batch(batch)
    assert (rep_o["iterations"] == rep_s["iterations"]).all()
    assert np.abs(rep_o["final_cost"] - rep_s["final_cost"]).max() < 1e-7 * rep_o["final_cost"].max()
    d = state_diffs(batch.state_array(), ref)
    assert d["para_Pose"] < 1e-7 and d["para_SpeedBias"] < 1e-5 and np.abs(batch.para_Feature - lam).max() < 1e-7, d


def _chained_windows_case(make_backend, nw=1, F=12, F0=8, iters=3, nthreads=4):
    """optimization() twice in a row, the way processImage() chains it: solve the previous window (frames -1..9), marginalize its oldest
    frame at the SOLVED states (estimator.cpp:1247-1376), solve the next window against that prior.  Same chain on the oracle."""
    cfg = small_cfg(max_batch=max(nw, 4), max_features=max(F, F0, 8), iters=iters)
    o, be = OracleBackend(cfg), make_backend(cfg)
    import ctypes as C
    out = []
    # Same eigen algorithm on both arms (cyclic Jacobi, the device's): this test pins the device chain against the restatement of the
    # SAME arithmetic.  What the choice of eigen-solver (the reference's tridiagonal QR vs Jacobi) does to a chained trajectory is
    # measured over >= 20 frames by tools/eig_study.py / tests/test_replay.py: the published poses move by
    # 1e-4 .. 4e-4 m under ANY rounding-level change of the marginalization, including two QR runs that only differ in summation order.
    o.set_eig_mode(1)
    try:
        _chained_windows_arms(o, be, cfg, nw, F, F0, nthreads, out, C)
    finally:
        o.set_eig_mode(0)
    _chained_windows_compare(out, nw)


def _chained_windows_arms(o, be, cfg, nw, F, F0, nthreads, out, C):
    for X in (o, be):
        batch = synth.generate_batch(nw, F, o, prior_features=F0, window0=91)
        pb = batch.prior_window
        rep_prev = (X.solve_batch(pb, nthreads=nthreads) if X is o else X.solve_batch(pb)).copy()
        X.marginalize(cfg, pb, batch, margin_old=True)
        before = (abi.WindowState * nw)()
        C.memmove(before, batch.states, C.sizeof(before))
        rep = (X.solve_batch(batch, nthreads=nthreads) if X is o else X.solve_batch(batch)).copy()
        # what the estimator publishes: the states after the yaw / position re-anchoring of double2vector (estimator.cpp:868-1005)
        anchored = [X.double2vector(before[w], batch.states[w]) for w in range(nw)]          # each arm through its OWN double2vector
        out.append((batch, rep_prev, rep, anchored))


def _chained_windows_compare(out, nw):
    (b0, rp0, r0, a0), (b1, rp1, r1, a1) = out
    assert (rp0["iterations"] == rp1["iterations"]).all() and (r0["iterations"] == r1["iterations"]).all()
    assert (r0["num_successful_steps"] == r1["num_successful_steps"]).all()
    for w in range(nw):
        A0, g0, x0 = prior_canonical(b0, w); A1, g1, x1 = prior_canonical(b1, w)
        assert np.abs(A0 - A1).max() < 1e-5 * np.abs(A0).max() and np.abs(g0 - g1).max() < 1e-4 * max(1.0, np.abs(g0).max())
        assert all(np.abs(x0[k][:7] - x1[k][:7]).max() < 1e-7 for k in x0)              # linearisation point = solved previous window
    # The eps-clamped eigen factoring of a gauge-deficient Hessian (|A| ~ 1e14 from near features; the eigenvalues that should be 0 are
    # rounding noise of either sign, far above eps = 1e-8) leaves implementation-dependent noise along the gauge directions of the
    # prior, which the next solve turns into a common drift of the raw poses: ~1e-5 m between the two Jacobi-based implementations
    # compared here, ~5e-4 m against the tridiagonal-QR eigen-solver of the reference's kind (oracle/sym_eig_qr.h).  double2vector's
    # yaw / position re-anchoring removes most of it.  Tolerances: the 1e-4 m bar of the path on the raw poses, 1e-5 on what the
    # estimator publishes.
    d = state_diffs(b1.state_array(), b0.state_array())
    assert d["para_Pose"] < 1e-4 and d["para_SpeedBias"] < 1e-4 and d["para_Ex_Pose"] < 1e-5, d
    for w in range(nw):
        for x, y in zip(a0[w], a1[w]):
            assert np.abs(np.asarray(x) - np.asarray(y)).max() < 1e-5
    assert np.abs(r0["final_cost"] - r1["final_cost"]).max() < 1e-4 * r0["final_cost"].max()


def test_chained_windows_match_oracle():
    _chained_windows_case(lambda cfg: sim_backend(cfg))


def test_host_buffer_pipeline_chunks(monkeypatch):
    """cerb_solve_batch packs / copies / solves in chunks on three compute lanes (here, through the test hook: 9 windows in chunks of 4, 4, 1, one lane
    each, four launches per chunk); windows with identical inputs must come back bit-identical whichever chunk / lane / workspace slice carried them.
    (Host-buffer path == resident path at 1024 windows is asserted on the GPU tier.)"""
    monkeypatch.setenv("CERB_TEST_CHUNK", "4")
    cfg = small_cfg(max_batch=16, max_features=8, iters=1)
    s = sim_backend(cfg)
    base = synth.generate_batch(3, 4, ob, with_prior=False, window0=140)
    big = synth.tile_batch(base, 9)
    rep = s.solve_batch(big)
    assert s.last_solve_stats()[1] == 4 * 3 + 1      # per chunk: pack, two prepare kernels, solve; + the unpack kernel of the download
    pose = big.state_array()["para_Pose"]
    assert not (pose[:3] == base.state_array()["para_Pose"]).all()                  # the solve moved the states
    for k in range(3, 9):
        assert (pose[k] == pose[k % 3]).all() and (big.para_Feature[k] == big.para_Feature[k % 3]).all()
    assert (rep["final_cost"][3:6] == rep["final_cost"][0:3]).all() and (rep["status"] == 0).all()


def test_host_buffer_pipeline_ramp(monkeypatch):
    """the shipped chunk schedule (first, first, 2 first, 4 first, ...; here first = 2 through the tuning knob: 9 windows -> 2, 2, 4, 1 on three lanes,
    lane 0 carries two chunks) against the single-chunk solve of the same batch: bit-identical states and reports"""
    cfg = small_cfg(max_batch=16, max_features=8, iters=1)
    s = sim_backend(cfg)
    base = synth.generate_batch(3, 4, ob, window0=145, prior_features=4)
    one = synth.tile_batch(base, 9); ramp = synth.tile_batch(base, 9)
    rep_one = s.solve_batch(one)
    assert s.last_solve_stats()[1] == 4 * 1 + 1
    monkeypatch.setenv("CERB_PIPE_FIRST", "2")
    rep_ramp = s.solve_batch(ramp)
    assert s.last_solve_stats()[1] == 4 * 4 + 1
    sa, sb = one.state_array(), ramp.state_array()
    for name in ("para_Pose", "para_SpeedBias", "para_LegBias", "para_Ex_Pose", "para_Td"):
        assert (sa[name] == sb[name]).all(), name
    assert (one.para_Feature == ramp.para_Feature).all()
    assert (rep_one["final_cost"] == rep_ramp["final_cost"]).all() and (rep_one["iterations"] == rep_ramp["iterations"]).all()


def test_bad_descriptor_in_a_later_chunk(monkeypatch):
    """a malformed window in the third chunk: the call fails with CERB_ERR_BAD_ARGUMENT after draining the chunks already in flight, and the handle
    stays usable"""
    from cerberus_b200 import lib as _lib
    monkeypatch.setenv("CERB_TEST_CHUNK", "2")
    cfg = small_cfg(max_batch=16, max_features=8, iters=1)
    s = sim_backend(cfg)
    base = synth.generate_batch(3, 4, ob, with_prior=False, window0=160)
    big = synth.tile_batch(base, 6)
    big.descs[5].n_features = cfg.max_features + 1
    with pytest.raises(_lib.CerbError) as e:
        s.solve_batch(big)
    assert e.value.code == abi.ERR_BAD_ARGUMENT
    big.descs[5].n_features = base.descs[2].n_features
    rep = s.solve_batch(big)
    assert (rep["status"] == 0).all() and (rep["final_cost"][3:] == rep["final_cost"][:3]).all()


def test_registered_host_buffers_take_the_zero_copy_path():
    _registered_buffers_case(sim_backend, 16, 9, 3)


def _registered_buffers_case(make_backend, max_batch, n, max_chunks, iters=1):
    """cerb_register_host_buffer: arrays inside registered memory are DMA'd straight out of the caller's buffers (ONE 2-D copy per array and
    pipeline chunk when the per-window arrays are uniformly strided), the others go through pinned staging.  Results are bit-identical."""
    cfg = small_cfg(max_batch=max_batch, max_features=8, iters=iters)
    s = make_backend(cfg)
    base = synth.generate_batch(3, 4, ob, window0=150, prior_features=4)
    big = synth.tile_batch(base, n)
    saved = big.copy_states()
    rep_a = s.solve_batch(big); out_a = np.frombuffer(big.states, dtype=np.uint8).copy(); lam_a = big.para_Feature.copy()
    ops_a, staged_a = s.last_upload_stats()
    assert staged_a > 0
    big.restore_states(saved)
    regs = s.register_batch(big)
    rep_b = s.solve_batch(big)
    ops_b, staged_b = s.last_upload_stats()
    assert staged_b == 0 and ops_b <= max_chunks * 10   # per chunk: descs, states, features, obs, para_Feature, preint head + tail, prior J, prior r
    assert (np.frombuffer(big.states, dtype=np.uint8) == out_a).all() and (big.para_Feature == lam_a).all() and (rep_a["final_cost"] == rep_b["final_cost"]).all()
    # irregular batch: one window without features, one without a prior -> per-window copies for those arrays, same results as staged
    big.restore_states(saved)
    big.descs[1].n_features = 0; big.descs[1].n_obs = 0; big.descs[4].prior.valid = 0
    rep_c = s.solve_batch(big); out_c = np.frombuffer(big.states, dtype=np.uint8).copy()
    assert s.last_upload_stats()[1] == 0
    s.unregister(regs)
    assert (rep_c["final_cost"][[0, 2, 3]] == rep_a["final_cost"][[0, 2, 3]]).all() and rep_c["final_cost"][1] != rep_a["final_cost"][1]


def test_marginalization_of_imu_only_windows():
    _imu_only_marginalization_case(sim_backend)


def _imu_only_marginalization_case(make_backend):
    """USE_LEG == 0 (estimator.cpp:1287-1297): the frame 0 -> 1 factor is IMUFactor <15,7,9,7,9>, there are no leg-bias blocks; the device
    path (IMU factor embedded in the 31-row kernels) against the oracle's MarginalizationInfo restatement with the plain IMUFactor."""
    cfg = small_cfg()
    s = make_backend(cfg)
    src = synth.generate_batch(2, 10, ob, use_leg=False, window0=61)
    a, b = synth.generate_batch(2, 10, ob, use_leg=False, window0=61), synth.generate_batch(2, 10, ob, use_leg=False, window0=61)
    ob.marginalize(cfg, src, a); s.marginalize(cfg, src, b)
    for w in range(2):
        A0, b0, x0 = prior_canonical(a, w); A1, b1, x1 = prior_canonical(b, w)
        assert A0.shape == A1.shape and set(x0) == set(x1) and not any(k[0] == abi.BLOCK_LEGBIAS for k in x1)
        assert np.abs(A0 - A1).max() < 1e-5 * np.abs(A0).max() and np.abs(b0 - b1).max() < 1e-4 * np.abs(b0).max()
